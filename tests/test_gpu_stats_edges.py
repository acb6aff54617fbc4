"""The error-statistics reducers at their edges, held to the exact reference (oracle/stats_exact.py: max|e| as
np.max(np.abs(e)), mean and ddof-0 std in integer arithmetic rounded once, NumPy's non-finite rules):

  K3   ensemble statistics (stats_small_kernel up to 2^17 elements, then the staged kernels), two-pass;
  K3x  K3 fused with the multi-GPU exchange, on one GPU (a world of one, and a world of two whose second slot
       is filled from the host), two-pass then Chan;
  K3p  per-run statistics of a device array (proc_stats_kernel), Welford then Chan;
  K9   IMU error statistics inside the generator, two-pass per stretch then Chan;
  K12  per-run process statistics of the Monte-Carlo kernel, one pass shifted by the first sample;
  K7   the same in the loosely-coupled filter's PROC form.

To isolate the reduction from the arithmetic that makes the errors, every reducer is compared with the exact
statistics of the errors the same launch stores: the arrays given to K3 / K3p, K1's series of the same K9
arguments, the histories K12 and K7 dump (dump_runs = R) against the same ref_nav.

Tolerances (stats_exact.assert_stats), derived from the algorithms:
  two-pass, Welford, Chan: every sum is a chain of at most DEPTH roundings (K3: <= 128 samples per thread,
    1024 thread partials, 128 block partials; K3p and K9: a handful of samples per thread, then 5 + 8 merges
    and a few tiles), so mean is within m = DEPTH eps max|e| and std within DEPTH eps std plus the mean's
    error: to second order, min(m, m^2 / std), after two passes (K3, K3x of one rank), to first order, m,
    after a Chan merge (K3p, K9, K3x of two ranks), whose mean_b - mean_a is rounded to eps max|e|;
  shifted one pass (K12, K7): the mean within (n + 2) eps max|e - e_first| + 2 eps max|e| (n sequential
    additions of the shifted errors); std within 1e-12 of itself on benign and offset data (the shift removes
    the offset), and within 1e-8 of itself when the first counted sample, the shift, lies 1e6 spreads from the
    rest (measured on an H100: 4.9e-9 at n = 2e5, 1.6e-10 at n = 2e4, at most 2.5e-13 on the other families);
  K3's path is pinned by the bits of its mean (test_k3_at_the_small_staged_switch);
  non-finite samples: NaN masks and infinities equal exactly, and every other run and column of the launch
    equals a launch without the non-finite sample bit for bit."""
import ctypes
import os

import numpy as np
import pytest

import stats_exact as sx
import oracle_np as onp
from conftest import load_golden, write_logged_dir

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')
EPS = sx.EPS
DEPTH_K3 = 2048
DEPTH_K3P = 64
DEPTH_K9 = 64
ATT_SLACK = 4 * EPS * np.pi          # the host's own rounding of the wrapped attitude error
MID_G = {'b': np.array([1e-5, -2e-5, 3e-6]), 'b_drift': np.full(3, 3.5 * np.pi / 180 / 3600),
         'b_corr': np.full(3, 100.0), 'arw': np.full(3, 0.25 * np.pi / 180 / 60)}
MID_A = {'b': np.array([2e-3, -1e-3, 5e-4]), 'b_drift': np.full(3, 5e-5), 'b_corr': np.full(3, 100.0),
         'vrw': np.full(3, 0.03 / 60)}


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _absmax(x, axis):
    """max|x| over the finite samples (the scale of the rounding errors)."""
    return np.where(np.isfinite(x), np.abs(x), 0.0).max(axis)


def _check(got, ref, x, axis, depth, what, std_from_mean):
    """A reduction whose chains of additions are at most `depth` long: mean within depth eps max|x|, std within
    depth eps std and the mean's error as std_from_mean says (stats_exact.assert_stats)."""
    sx.assert_stats(got, ref, depth * EPS * _absmax(x, axis), depth * EPS, what, std_from_mean)


def _family(rng, kind, n, nc):
    """[n, nc] samples: benign (Gaussian, moderate offsets), offset-dominated D + sigma z with D / sigma from 1e3
    to 1e9 across the columns, the first sample far from the rest, or a constant."""
    z = rng.standard_normal((n, nc))
    if kind == 'benign':
        return z * np.logspace(-3, 2, nc) + np.linspace(-2.0, 2.0, nc)
    if kind == 'offset':
        ratio = np.logspace(3, 9, nc) if nc > 1 else np.array([1e9])
        return 5.0 + (5.0 / ratio) * z
    if kind == 'outlier':
        x = 1e3 + 1e-3 * z
        x[0] = 0.0
        return x
    if kind == 'constant':
        return np.tile(np.linspace(-0.1, 0.3, nc), (n, 1))
    raise ValueError(kind)


# ---- K3 ----------------------------------------------------------------------------------------------------
def _k3_shapes():
    out = []
    for nc in (1, 7, 27, 32):
        lo = (1 << 17) // nc
        runs = {lo, lo + 1} | ({lo - 1} if lo * nc == 1 << 17 else set())
        out += [(r, nc) for r in sorted(runs)]
    return out


def _k3_mean_small(x):
    """The mean stats_small_kernel computes, in its order of additions: thread t of (1024 / nc) nc sums elements
    t, t + threads, ... of the flat [runs][nc] array; thread c < nc then sums the partials c, c + nc, ..."""
    runs, nc = x.shape
    threads = (1024 // nc) * nc
    flat = x.reshape(-1)
    k = -(-flat.size // threads)
    pad = np.zeros(k * threads)
    pad[:flat.size] = flat                       # a thread past the end adds nothing; + 0.0 is exact
    acc = np.zeros(threads)
    for i in range(k):
        acc = acc + pad[i * threads:(i + 1) * threads]
    s = np.zeros(nc)
    for row in acc.reshape(threads // nc, nc):
        s = s + row
    return s / runs


def _k3_mean_staged(x):
    """The mean of the staged kernels (err_stage1/2_kernel, stats_mean_kernel), in their order: 32 nc threads
    per block, min(128, ceil(total / threads)) blocks, grid-stride sums per thread, the block's partials of
    column c in thread order, then the blocks in order."""
    runs, nc = x.shape
    threads = nc * (32 if 1024 // nc >= 32 else 1024 // nc)
    flat = x.reshape(-1)
    grid = min(128, max(1, -(-flat.size // threads)))
    stride = grid * threads
    k = -(-flat.size // stride)
    pad = np.zeros(k * stride)
    pad[:flat.size] = flat
    acc = np.zeros(stride)
    for i in range(k):
        acc = acc + pad[i * stride:(i + 1) * stride]
    part = acc.reshape(grid, threads // nc, nc)
    blocks = np.zeros((grid, nc))
    for r in range(threads // nc):
        blocks = blocks + part[:, r, :]
    s = np.zeros(nc)
    for b in range(grid):
        s = s + blocks[b]
    return s / runs


@pytest.mark.parametrize('runs,nc', _k3_shapes())
def test_k3_at_the_small_staged_switch(eng, runs, nc):
    """runs * ncomp just below, at and above 2^17, where K3 switches from one block to the staged kernels.  Both
    paths are accurate, so the path is pinned by its bits: the mean equals, bit for bit, a float64 restatement
    of the order of additions of the path that must run (the one block up to 2^17 elements, the staged kernels
    above), and the data make the two orders differ.  Up to 2^17 it also equals K3x's local pass (the same
    one-block order) bit for bit."""
    x = _family(np.random.default_rng(runs), 'offset', runs, nc)
    got = eng.error_stats(_dev(x)).cpu().numpy()
    _check(got, sx.stats(x), x, 0, DEPTH_K3, 'K3 %dx%d' % (runs, nc), 'second')
    small, staged = _k3_mean_small(x), _k3_mean_staged(x)
    assert (small != staged).any(), 'the data do not tell the two orders apart'
    one_block = runs * nc <= 1 << 17
    assert np.array_equal(got[1], small if one_block else staged), 'K3 took the other path'
    if one_block and 3 * nc + 2 <= XSLOT:
        assert np.array_equal(_k3x(eng, x, 1)[:2], got[:2])


@pytest.mark.parametrize('kind', ['benign', 'offset', 'outlier', 'constant'])
@pytest.mark.parametrize('runs', [1, 2, 3, 1000])
def test_k3_families(eng, kind, runs):
    """Fewer elements than one block, one and two runs, and the data families."""
    for nc in (1, 9, 32):
        x = _family(np.random.default_rng(runs * 100 + nc), kind, runs, nc)
        got = eng.error_stats(_dev(x)).cpu().numpy()
        _check(got, sx.stats(x), x, 0, DEPTH_K3, 'K3 %s %d' % (kind, runs), 'second')


def _inject(x, what, at):
    """x with one NaN / +inf / -inf at index `at`, or the column at[-1] all NaN ('column')."""
    y = x.copy()
    if what == 'column':
        y[(slice(None),) * (y.ndim - 1) + (at[-1],)] = np.nan
    else:
        y[at] = {'nan': np.nan, '+inf': np.inf, '-inf': -np.inf}[what]
    return y


@pytest.mark.parametrize('what', ['nan', '+inf', '-inf', 'column'])
@pytest.mark.parametrize('runs,nc', [(37, 9), (1 << 17, 1), ((1 << 17) // 9 + 1, 9)])
def test_k3_non_finite(eng, runs, nc, what):
    """One non-finite error in one column (or one column all NaN), on both paths: that column is NaN / inf as
    NumPy's, every other column equals the launch without it bit for bit."""
    x = _family(np.random.default_rng(5), 'benign', runs, nc)
    c = nc // 2
    y = _inject(x, what, (runs // 3, c))
    clean = eng.error_stats(_dev(x)).cpu().numpy()
    got = eng.error_stats(_dev(y)).cpu().numpy()
    _check(got, sx.stats(y), y, 0, DEPTH_K3, 'K3 %s' % what, 'second')
    others = np.arange(nc) != c
    assert np.array_equal(got[:, others], clean[:, others])
    with np.errstate(invalid='ignore'):
        np_ = np.stack([np.max(np.abs(y), 0), np.average(y, 0), np.std(y, 0)])
    assert np.array_equal(np.isnan(got), np.isnan(np_)) and np.array_equal(np.isinf(got), np.isinf(np_))


# ---- K3x on one GPU ----------------------------------------------------------------------------------------
XSLOT = 32             # kXchgSlot: doubles per (parity, source rank): max, mean, std [nc each], count, flag


def _k3x(eng, x, world, peer_stats=None, seq=1):
    """stats_exchange_kernel as rank 0 of `world` on this GPU.  world 2: rank 1's slot of this rank's window is
    filled from the host with peer_stats = (n, max, mean, std) and its flag = seq before the launch, so the
    kernel's wait ends at once and it runs its Chan merge on one device."""
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    nc = x.shape[1]
    wins = [torch.zeros(2 * world * XSLOT, dtype=torch.float64, device='cuda') for _ in range(world)]
    par = seq & 1
    if world == 2:
        n, mx, mean, std = peer_stats
        slot = np.zeros(XSLOT)
        slot[0:nc], slot[nc:2 * nc], slot[2 * nc:3 * nc], slot[3 * nc] = mx, mean, std, float(n)
        slot.view(np.uint64)[XSLOT - 1] = seq
        off = (par * world + 1) * XSLOT
        wins[0][off:off + XSLOT] = torch.from_numpy(slot).cuda()
        assert int(wins[0][off + XSLOT - 1:off + XSLOT].cpu().numpy().view(np.uint64)[0]) == seq
    ptrs = (ctypes.c_uint64 * world)(*[w.data_ptr() for w in wins])
    err = _dev(x)
    out = torch.zeros((3, nc), dtype=torch.float64, device='cuda')
    flag = torch.zeros(1, dtype=torch.int32, device='cuda')
    _lib.check(lib.b2ins_error_stats_exchange_f64(
        x.shape[0], nc, ctypes.c_void_p(err.data_ptr()), 0, world, ptrs, seq, ctypes.c_void_p(out.data_ptr()),
        ctypes.c_void_p(flag.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert int(flag.item()) == 0, 'the exchange timed out'
    return out.cpu().numpy()


@pytest.mark.parametrize('kind', ['benign', 'offset', 'outlier'])
def test_k3x_world_of_one(eng, kind):
    for runs, nc in ((1, 9), (2, 9), (1000, 9), ((1 << 17) // 10, 10), (77, 1)):
        x = _family(np.random.default_rng(runs), kind, runs, nc)
        got = _k3x(eng, x, 1)
        _check(got, sx.stats(x), x, 0, DEPTH_K3, 'K3x %s %d' % (kind, runs), 'second')


def test_k3x_no_runs_is_nan(eng):
    """Every shard empty: the statistics of no samples are NaN (a world of one with no runs)."""
    assert np.isnan(_k3x(eng, np.zeros((0, 9)), 1)).all()


@pytest.mark.parametrize('case', ['benign', 'offset', 'nan_here', 'nan_there', 'inf_here', 'inf_both_signs'])
def test_k3x_merge_of_two(eng, case):
    """Rank 0's shard on the device, rank 1's statistics from the host: the merge equals dist.merge_stats and
    the exact statistics of the union, NaN and inf included."""
    from gnss_ins_sim_b200 import dist
    rng = np.random.default_rng(9)
    nc = 9
    a = _family(rng, 'offset' if case == 'offset' else 'benign', 300, nc)
    b = _family(rng, 'offset' if case == 'offset' else 'benign', 211, nc) + 0.25
    if case == 'nan_here':
        a[17, 2] = np.nan
    elif case == 'nan_there':
        b[5, 4] = np.nan
    elif case == 'inf_here':
        a[0, 6] = np.inf
    elif case == 'inf_both_signs':
        a[3, 7], b[8, 7] = np.inf, -np.inf
    with np.errstate(invalid='ignore'):
        sb = (b.shape[0], np.max(np.abs(b), 0), np.average(b, 0), np.std(b, 0))
    got = _k3x(eng, a, 2, sb)
    sa = eng.error_stats(_dev(a)).cpu().numpy()
    host, n = dist.merge_stats([(a.shape[0], sa[0], sa[1], sa[2]), sb])
    assert n == a.shape[0] + b.shape[0]
    u = np.concatenate([a, b])
    _check(got, sx.stats(u), u, 0, DEPTH_K3, 'K3x ' + case, 'first')
    assert np.array_equal(np.isnan(got), np.isnan(host)) and np.array_equal(got[np.isinf(host)],
                                                                            host[np.isinf(host)])
    fin = np.isfinite(host)
    assert np.all(np.abs(got - host)[fin] <= 1e-12 * np.maximum(np.abs(host), 1e-300)[fin] + 1e-300)


# ---- K3p ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('nc', range(1, 9))
def test_k3p_shapes(eng, nc):
    """m around one CTA's 256 rows, start on and beside the row-stride boundaries and on the last row, every
    nc; three runs, the columns from benign to offset-dominated."""
    rng = np.random.default_rng(nc)
    for m in (1, 255, 256, 257, 513):
        for start in sorted({s for s in (0, 255, 256, m - 1) if s < m}):
            for kind in ('benign', 'offset', 'outlier'):
                x = np.stack([_family(rng, kind, m, nc) for _ in range(3)])
                ref = rng.standard_normal((m, nc)) * 1e-9 if kind != 'benign' else np.zeros((m, nc))
                end, proc = eng.proc_stats(_dev(x + ref), _dev(ref), start)
                e = (x + ref) - ref                          # the kernel's own subtraction
                what = 'K3p m %d start %d nc %d %s' % (m, start, nc, kind)
                assert np.array_equal(end.cpu().numpy(), e[:, -1]), what
                st = proc.cpu().numpy()
                _check(st, sx.per_run(e, start), e[:, start:], 1, DEPTH_K3P, what, 'first')
                if m - start == 1:
                    assert np.array_equal(st[:, 1], e[:, -1]) and np.all(st[:, 2] == 0.0)


@pytest.mark.parametrize('what', ['nan', '+inf', '-inf', 'column', 'nan_before_start'])
def test_k3p_non_finite(eng, what):
    rng = np.random.default_rng(3)
    R_, m, nc, start = 4, 700, 6, 100
    x = rng.standard_normal((R_, m, nc)) + 2.0
    ref = np.zeros((m, nc))
    at = (2, 50 if what == 'nan_before_start' else 400, 3)
    y = _inject(x, 'nan' if what == 'nan_before_start' else what, at)
    if what == 'column':
        y = x.copy()
        y[2, :, 3] = np.nan
    _, clean = eng.proc_stats(_dev(x), _dev(ref), start)
    _, got = eng.proc_stats(_dev(y), _dev(ref), start)
    got, clean = got.cpu().numpy(), clean.cpu().numpy()
    _check(got, sx.per_run(y, start), y[:, start:], 1, DEPTH_K3P, 'K3p ' + what, 'first')
    keep = np.ones((R_, nc), dtype=bool)
    if what != 'nan_before_start':
        keep[2, 3] = False
        assert not np.isfinite(got[2, :, 3]).all()
    assert np.array_equal(got.transpose(0, 2, 1)[keep], clean.transpose(0, 2, 1)[keep])


# ---- K9 ----------------------------------------------------------------------------------------------------
def _k9(eng, ref_g, ref_a, R_, start, seed=3):
    rg, ra = _dev(ref_g), _dev(ref_a)
    end, proc = eng.imu_err_stats(100.0, R_, rg, ra, MID_G, MID_A, seed, run_offset=2, stats_start=start)
    gyro, accel = eng.imu_noise(100.0, R_, rg, ra, MID_G, MID_A, seed, run_offset=2)
    e = torch.cat([accel - ra[None], gyro - rg[None]], dim=2).cpu().numpy()
    return end.cpu().numpy(), proc.cpu().numpy(), e


@pytest.mark.parametrize('n', [895, 896, 897, 896 * 3 + 1])
def test_k9_tile_edges(eng, n):
    """n around 896-sample tiles; start 0, inside the first thread's 7-sample stretch, on a thread boundary, on
    a tile boundary and on the last sample; the errors of K1's series of the same call."""
    rng = np.random.default_rng(n)
    ref_g, ref_a = rng.standard_normal((n, 3)) * 0.3, rng.standard_normal((n, 3)) * 3.0 + [0.0, 0.0, -9.8]
    for start in sorted({s for s in (0, 3, 7, 896, n - 1) if s < n}):
        end, proc, e = _k9(eng, ref_g, ref_a, 5, start)
        assert np.array_equal(end, e[:, -1])
        _check(proc, sx.per_run(e, start), e[:, start:], 1, DEPTH_K9, 'K9 n %d start %d' % (n, start), 'first')


@pytest.mark.parametrize('what', ['accel_nan', 'gyro_nan', 'accel_inf', 'nan_before_start'])
def test_k9_non_finite_reference_row(eng, what):
    """One non-finite value in ref_accel or ref_gyro (meas = ref + noise, so e = NaN there for NaN and inf):
    that column is NaN in every run; a NaN before the start does not count; the other columns, and the column
    whose NaN lies before the start, equal the launch without it bit for bit."""
    n, R_, start = 2000, 5, 300
    rng = np.random.default_rng(1)
    ref_g, ref_a = rng.standard_normal((n, 3)) * 0.3, rng.standard_normal((n, 3)) * 3.0
    g2, a2 = ref_g.copy(), ref_a.copy()
    col = {'accel_nan': 1, 'gyro_nan': 5, 'accel_inf': 0, 'nan_before_start': 4}[what]
    row = 100 if what == 'nan_before_start' else 1234
    tgt, c = (a2, col) if col < 3 else (g2, col - 3)
    tgt[row, c] = np.inf if what == 'accel_inf' else np.nan
    _, clean, _ = _k9(eng, ref_g, ref_a, R_, start)
    end, proc, e = _k9(eng, g2, a2, R_, start)
    _check(proc, sx.per_run(e, start), e[:, start:], 1, DEPTH_K9, 'K9 ' + what, 'first')
    others = np.arange(6) != col
    assert np.array_equal(proc[:, :, others], clean[:, :, others])
    if what == 'nan_before_start':
        assert np.array_equal(proc, clean)
    else:
        assert np.isnan(proc[:, :, col]).all()


def test_k9_nan_in_a_later_time_segment(eng):
    """3 runs x 300 000 samples take the time-segmented path: a NaN ref_accel value inside the third segment
    reaches err_stats_fold_kernel as one segment's NaN partial.  That column is NaN in every run; the other
    columns equal the launch without it bit for bit, and the end-point errors are K1's."""
    from test_gpu_sensor_stats import _seg_len
    n, R_, start = 300000, 3, 100
    seg = _seg_len(n, R_)
    assert -(-n // seg) >= 3, 'not segmented: %d samples per segment' % seg
    rng = np.random.default_rng(6)
    ref_g, ref_a = rng.standard_normal((n, 3)) * 0.3, rng.standard_normal((n, 3)) * 3.0
    a2 = ref_a.copy()
    a2[2 * seg + 5, 1] = np.nan
    _, clean, _ = _k9(eng, ref_g, ref_a, R_, start)
    end, proc, e = _k9(eng, ref_g, a2, R_, start)
    assert np.array_equal(end, e[:, -1])
    assert np.isnan(proc[:, :, 1]).all()
    others = np.arange(6) != 1
    assert np.array_equal(proc[:, :, others], clean[:, :, others])


# ---- K12 ---------------------------------------------------------------------------------------------------
def _static_case(n):
    """The first sample of the 90-degree turn (ref_frame 1) held for n samples: the state drifts away from its
    start, and the errors against ref_nav are whatever ref_nav makes them (it enters nothing but the errors)."""
    g = load_golden('traj_90deg_turn_100hz_rf1.npz')
    nav0 = np.concatenate([g['ref_att'][0], g['ref_pos'][0], g['ref_vel'][0]])
    return (np.tile(g['ref_gyro'][0], (n, 1)), np.tile(g['ref_accel'][0], (n, 1)), np.tile(nav0, (n, 1)),
            g['ini'])


def _k12(eng, rg, ra, nav, ini, R_, start, lanes, seed=7):
    from gnss_ins_sim_b200 import imu_model
    imu = imu_model.IMU(accuracy='mid-accuracy', axis=6, gps=False)
    ini = np.atleast_2d(ini)
    cfg = eng.make_mc_config(1, 100.0, rg.shape[0], R_, seed, imu.gyro_err, imu.accel_err, ini.shape[0], 9,
                             lanes_per_run=lanes, stats_start=start, dump_runs=R_)
    res = eng.mc_free_integration(cfg, _dev(rg), _dev(ra), _dev(nav), _dev(ini), dump_nav=True)
    att, pos, vel = (t.cpu().numpy() for t in (res.att, res.pos, res.vel))
    with np.errstate(invalid='ignore'):
        e = np.concatenate([onp.angle_range_pi(att - nav[None, :, 0:3]), pos - nav[None, :, 3:6],
                            vel - nav[None, :, 6:9]], axis=2)
    return res.proc_stats.cpu().numpy(), e


def _check_one_pass(ps, e, start, rel, what):
    """The shifted one pass: mean within stats_exact.one_pass_mean_err, std within `rel` of itself (the shift has
    removed the offset; the mean's rounding is in it).  pos / vel: the same errors, max bit for bit; attitude:
    the host's wrap may round differently."""
    ex = sx.per_run(e, start)
    me = sx.one_pass_mean_err(e, start)
    sx.assert_stats(ps[:, :, 3:], ex[:, :, 3:], me[:, 3:], rel, what + ' pos/vel', 'none')
    sx.assert_stats(ps[:, :, :3], ex[:, :, :3], me[:, :3], rel, what + ' att', 'none', max_exact=False,
                    abs_slack=ATT_SLACK)
    fin = np.isfinite(ex) & (ex[:, 2:3] > 0)
    worst = np.abs(ps - ex)[:, 2][fin[:, 2]] / ex[:, 2][fin[:, 2]]
    print(what, 'worst relative std error %.2e' % (worst.max() if worst.size else 0.0))


@pytest.mark.parametrize('lanes', [1, 2, 4, 8, 16, 32])
def test_k12_every_lane_group(eng, lanes):
    """37 runs (not a multiple of any CTA's runs), benign and offset-dominated errors (position and velocity of
    ref_nav moved 1e6 times the errors' spread away), start 0, mid-series and the last sample."""
    n, R_ = 3000, 37
    rg, ra, nav, ini = _static_case(n)
    _, e0 = _k12(eng, rg, ra, nav, ini, R_, 0, lanes)
    spread = np.std(e0, axis=1).max(0)
    for kind in ('benign', 'offset'):
        nv = nav.copy()
        if kind == 'offset':
            nv[:, 3:9] -= 1e6 * spread[3:9]
        for start in (0, 1234, n - 1):
            ps, e = _k12(eng, rg, ra, nv, ini, R_, start, lanes)
            _check_one_pass(ps, e, start, 1e-12, 'K12 lanes %d %s start %d' % (lanes, kind, start))
            if start == n - 1:
                assert np.all(ps[:, 2] == 0.0)


def test_k12_first_sample_far_from_the_rest(eng):
    """The shift is the first counted sample; here it lies ~1e6 standard deviations from the others, where the
    one-pass variance loses the most (n up to 2e5): within 1e-8 relative."""
    for n in (20000, 200000):
        rg, ra, nav, ini = _static_case(n)
        start = 10
        nv = nav.copy()
        ps0, e0 = _k12(eng, rg, ra, nv, ini, 3, start, 1)
        spread = np.std(e0[:, start:], axis=1).max(0)
        nv[start, 3:9] += 1e6 * spread[3:9]
        ps, e = _k12(eng, rg, ra, nv, ini, 3, start, 1)
        _check_one_pass(ps, e, start, 1e-8, 'K12 outlier n %d' % n)
        assert np.array_equal(ps[:, :, :3], ps0[:, :, :3])


@pytest.mark.parametrize('what', ['nan', '+inf', '-inf', 'nan_before_start', 'nan_first', 'inf_first', 'nan_yaw'])
def test_k12_non_finite(eng, what):
    """One non-finite value in one ref_nav column (every run's error there), at the start, before it, or a NaN
    initial yaw in run 10 (its attitude goes NaN like the reference's): NaN and inf where NumPy has them, the
    rest of the launch unchanged bit for bit."""
    n, R_, start = 2000, 37, 200
    rg, ra, nav, ini = _static_case(n)
    ini_r = np.tile(ini, (R_, 1))
    clean, _ = _k12(eng, rg, ra, nav, ini_r, R_, start, 8)
    nv, ir = nav.copy(), ini_r.copy()
    col = 4
    if what == 'nan_yaw':
        ir[10, 6] = np.nan
    else:
        row = {'nan_before_start': 50, 'nan_first': start, 'inf_first': start}.get(what, 1500)
        nv[row, col] = {'+inf': np.inf, '-inf': -np.inf, 'inf_first': np.inf}.get(what, np.nan)
    ps, e = _k12(eng, rg, ra, nv, ir, R_, start, 8)
    _check_one_pass(ps, e, start, 1e-12, 'K12 ' + what)
    keep = np.ones((R_, 9), dtype=bool)
    if what == 'nan_yaw':
        keep[10] = False
        assert np.isnan(ps[10]).any()
    elif what != 'nan_before_start':
        keep[:, col] = False
        assert not np.isfinite(ps[:, :, col]).all()
    assert np.array_equal(ps.transpose(0, 2, 1)[keep], clean.transpose(0, 2, 1)[keep])


# ---- K7 ----------------------------------------------------------------------------------------------------
def _k7(eng, nav, start, align=None, vis=None):
    from test_gpu_ekf_proc import _turn_case, _launch, _imu, R, R0
    t, g, nav0, idx = _turn_case()
    if vis is not None:
        g['gps_visibility'] = vis(g['gps_visibility'])
    res = _launch(eng, t, g, nav0 if nav is None else nav, idx, _imu(), R, run_offset=R0, proc_start=start,
                  dump_runs=R, align=align)
    nv = nav0 if nav is None else nav
    att, pos, vel = (x.cpu().numpy() for x in (res.att, res.pos, res.vel))
    with np.errstate(invalid='ignore'):
        e = np.concatenate([onp.angle_range_pi(att - nv[None, :, 0:3]), pos - nv[None, :, 3:6],
                            vel - nv[None, :, 6:9]], axis=2)
    return res.proc_stats.cpu().numpy(), e, nav0


@pytest.mark.parametrize('start', [0, 777, -1])
def test_k7_thirteen_runs(eng, start):
    """13 runs (two CTAs of 8, the second ragged), the last sample as start included."""
    n = load_golden('traj_90deg_turn_100hz_rf0.npz')['ref_gyro'].shape[0]
    s = start if start >= 0 else n - 1
    ps, e, _ = _k7(eng, None, s)
    _check_one_pass(ps, e, s, 1e-12, 'K7 start %d' % s)
    if s == n - 1:
        assert np.all(ps[:, 2] == 0.0)


def test_k7_first_sample_far_from_the_rest(eng):
    """Position and velocity of the first counted sample 1e6 of their spread away from the others."""
    start = 500
    ps0, e0, nav = _k7(eng, None, start)
    spread = np.std(e0[:, start:], axis=1).max(0)
    nv = nav.copy()
    nv[start, 3:9] += 1e6 * spread[3:9]
    ps, e, _ = _k7(eng, nv, start)
    _check_one_pass(ps, e, start, 1e-8, 'K7 outlier')
    assert np.array_equal(ps[:, :, :3], ps0[:, :, :3])


@pytest.mark.parametrize('what', ['nan', '+inf', '-inf', 'nan_before_start', 'nan_first', 'inf_first'])
def test_k7_non_finite(eng, what):
    """ref_nav enters K7's PROC statistics and its consistency record only, not the filter: one non-finite
    ref_nav value makes that column of every run NaN / inf as NumPy's, and leaves the rest bit for bit."""
    start, col = 400, 7
    clean, _, nav = _k7(eng, None, start)
    nv = nav.copy()
    row = {'nan_before_start': 100, 'nan_first': start, 'inf_first': start}.get(what, 900)
    nv[row, col] = {'+inf': np.inf, '-inf': -np.inf, 'inf_first': np.inf}.get(what, np.nan)
    ps, e, _ = _k7(eng, nv, start)
    _check_one_pass(ps, e, start, 1e-12, 'K7 ' + what)
    others = np.arange(9) != col
    assert np.array_equal(ps[:, :, others], clean[:, :, others])
    if what == 'nan_before_start':
        assert np.array_equal(ps, clean)
    else:
        assert not np.isfinite(ps[:, :, col]).all()


def test_k7_without_a_fix_is_nan(eng):
    """An aligned filter that never sees a GPS row has no samples to count: max, mean and std are NaN (the
    statistics of no samples), as include/b2ins.h states."""
    ps, _, _ = _k7(eng, None, 100, align=('gps', 0.0), vis=np.zeros_like)
    assert ps.shape[1:] == (3, 9) and np.isnan(ps).all()


# ---- through Sim ---------------------------------------------------------------------------------------------
def test_sim_logged_run_with_a_nan_gyro_row(eng, tmp_path):
    """A logged-data directory of two runs, the second with one NaN gyro row, and FreeIntegration: the process
    statistics of that run and the end-point statistics over the runs are NaN exactly where NumPy's statistics
    of the get_data histories are; the first run's are those of a directory without the NaN run.  For logged
    data Sim takes the per-run process statistics on the host, so only the end-point half reaches a kernel
    (K3 on end_err); test_sim_generated_run_with_a_nan_initial_yaw takes the per-run half through K12."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    g = load_golden('logged_bosch.npz')
    d = write_logged_dir(str(tmp_path / 'two'), g)
    one = write_logged_dir(str(tmp_path / 'one'), g)
    gyro = g['gyro'].copy()
    gyro[len(gyro) // 2, 1] = np.nan
    np.savetxt(os.path.join(d, 'gyro-1.csv'), gyro * 180.0 / np.pi, delimiter=',', comments='',
               header='gyro_x (deg/s),gyro_y (deg/s),gyro_z (deg/s)', fmt='%.18e')
    np.savetxt(os.path.join(d, 'accel-1.csv'), g['accel'], delimiter=',', comments='',
               header='accel_x (m/s^2),accel_y (m/s^2),accel_z (m/s^2)', fmt='%.18e')
    sims = []
    for path, runs in ((d, 2), (one, 1)):
        s = Sim([100.0, 0.0, 0.0], path, ref_frame=0, imu=None,
                algorithm=FreeIntegration(g['ini'], earth_rot=False))
        s.run(runs)
        sims.append(s)
    sim, ref_sim = sims
    att = sim.get_data(['att_euler'])[0]
    with np.errstate(invalid='ignore'):      # against the directory's all-zero reference attitude
        e = [onp.angle_range_pi(att['algo0_%d' % r]) for r in (0, 1)]
    assert np.isnan(e[1]).any() and np.isfinite(e[0]).all()
    ps = sim.get_error_stats('att_euler', 0)
    for r in (0, 1):
        with np.errstate(invalid='ignore'):
            np_ = np.stack([np.max(np.abs(e[r]), 0), np.average(e[r], 0), np.std(e[r], 0)])
        got = np.stack([np.asarray(ps[k]['algo0_%d' % r], dtype=np.float64) for k in ('max', 'avg', 'std')])
        assert np.array_equal(np.isnan(got), np.isnan(np_)), (r, got, np_)
    base = ref_sim.get_error_stats('att_euler', 0)
    for k in ('max', 'avg', 'std'):
        assert np.array_equal(np.asarray(ps[k]['algo0_0']), np.asarray(base[k]['algo0_0']))
    end = sim.get_error_stats('att_euler', -1)
    last = np.stack([x[-1] for x in e])
    with np.errstate(invalid='ignore'):
        np_ = np.stack([np.max(np.abs(last), 0), np.average(last, 0), np.std(last, 0)])
    got = np.stack([np.asarray(end[k], dtype=np.float64) for k in ('max', 'avg', 'std')])
    assert np.isnan(np_).any() and np.array_equal(np.isnan(got), np.isnan(np_)), (got, np_)


def test_sim_generated_run_with_a_nan_initial_yaw(eng):
    """Generated Monte-Carlo runs through Sim and FreeIntegration with two initial-state sets, the second with a
    NaN yaw (run 1 uses it, runs 0 and 2 the first): get_error_stats('att_euler', 0) -- K12's per-run process
    statistics -- and the end-point statistics over the runs (K3) are NaN exactly where NumPy's statistics of
    the get_data histories are, and equal them to 1e-9 elsewhere."""
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    g = load_golden('traj_90deg_turn_100hz_rf0.npz')
    ini = np.stack([g['ini'], g['ini']], axis=1)
    ini[6, 1] = np.nan
    imu = imu_model.IMU(accuracy='mid-accuracy', axis=6, gps=False)
    sim = Sim([100.0, 0.0, 0.0], os.path.join(os.path.dirname(__file__), 'golden', 'motion_def-90deg_turn.csv'),
              ref_frame=0, imu=imu, algorithm=FreeIntegration(ini), seed=5)
    sim.run(3)
    att = sim.get_data(['att_euler'])[0]
    ref = sim.data['ref_att_euler']
    with np.errstate(invalid='ignore'):
        e = [onp.angle_range_pi(att['algo0_%d' % r] - ref) for r in range(3)]
    assert np.isnan(e[1]).any() and np.isfinite(e[0]).all() and np.isfinite(e[2]).all()

    def numpy_stats(x, axis):
        with np.errstate(invalid='ignore'):
            return np.stack([np.max(np.abs(x), axis), np.average(x, axis), np.std(x, axis)])

    def check(got, want, what):
        assert np.array_equal(np.isnan(got), np.isnan(want)), (what, got, want)
        fin = np.isfinite(want)
        assert np.all(np.abs(got - want)[fin] <= 1e-9 * np.maximum(np.abs(want)[fin], 1e-6)), what

    ps = sim.get_error_stats('att_euler', 0)
    for r in range(3):
        got = np.stack([np.asarray(ps[k]['algo0_%d' % r], dtype=np.float64) for k in ('max', 'avg', 'std')])
        check(got, numpy_stats(e[r], 0), 'run %d' % r)
    assert np.isnan(np.asarray(ps['max']['algo0_1'], dtype=np.float64)).all()
    end = sim.get_error_stats('att_euler', -1)
    got = np.stack([np.asarray(end[k], dtype=np.float64) for k in ('max', 'avg', 'std')])
    want = numpy_stats(np.stack([x[-1] for x in e]), 0)
    assert np.isnan(want).any()
    check(got, want, 'end point')
