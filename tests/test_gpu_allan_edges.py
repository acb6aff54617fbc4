"""K4, the reference estimator allan.allan_var, held to the exact reference (oracle/allan_exact.py) on every
front end of allan_launch, at the shapes, tau grids, data and non-finite samples where it can go wrong.

Error bound.  K4 does not round like the reference: it sums level by level.  For a tau m = j 10^k with nb
bins, the bound below follows K4's own order of operations (u = 2^-53, g_p = p u / (1 - p u)):
  * decade sums S_{k+1}[i], of ten S_k (S_0 = x): each element minus the tile's offset o, a tree of ten, plus
    10 o; the stored value carries E_{k+1}[i] <= sum E_k + g_11 (sum |S_k - o| + 10 |o| + |S_{k+1}|);
  * a successive difference d of two clusters of j elements of level k, offset-subtracted, summed and
    subtracted: |d^ - d| <= e_d = sum over both bins of E_k + g_{j+1} (sum |S_k - o| + |d|);
  * the square, by FMA into a chain: |d^2 - d^2| <= e_d (2 |d| + e_d);
  * the folds (a thread's chain of <= 30, a 5-step warp butterfly, <= 16 warps, then per chunk lane
    ceil(chunks / 32) and a 5-step butterfly, or the one-CTA rest kernel's ceil(nb / 512) + 5 + 16) of
    depth D: g_D of the sum of the terms; then three roundings in 0.5 / (nb - 1) * (s / (m m)).
The offset o is 0 at level 0 of the tiled front ends, the tile's first element at their levels >= 1 (the
halo's first element for a chunk > 0) and the level's first element in the rest kernel; 0 where that
element is not finite.  |K4 - exact| <= bound is asserted for every finite tau; a non-finite tau must be
of the exact reference's class (NaN or +inf)."""
import numpy as np
import pytest

import allan_exact as ae
import oracle_np as onp
from conftest import write_logged_dir, load_golden

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

U = 2.0 ** -53
CH = 5040
WORST = {}          # front end -> worst err / bound, printed at the end of the module


def _g(p):
    return p * U / (1.0 - p * U)


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


@pytest.fixture(scope='module')
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nK4 worst |K4 - exact| / bound per front end: ' +
          ', '.join('%s %.3g' % kv for kv in sorted(WORST.items())))


# ---------------------------------------------------------------------------------------------------------
# the bound
# ---------------------------------------------------------------------------------------------------------
def _offsets(s, rest):
    """The offset each element's tile subtracts (per element of the level), 0 where not finite."""
    if rest:
        o = np.full(len(s), s[0] if len(s) else 0.0)
    else:
        c = np.arange(len(s)) // CH
        o = s[np.maximum(c * CH - 9, 0)]
    return np.where(np.isfinite(o), o, 0.0)


def k4_bound(x, fs, exact):
    """Per tau, the bound on |K4 - exact| described in the module docstring."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    mult = onp.allan_multipliers(n, fs)
    out = np.zeros(len(mult))
    s, E = x, np.zeros(n)
    with np.errstate(invalid='ignore', over='ignore'):
        for k in range(12):
            L = len(s)
            rest = L <= CH
            o = _offsets(s, rest) if (k > 0 or rest) else np.zeros(L)
            chunks = 1 if rest else -(-L // CH)
            for i, m in enumerate(mult):
                if m // 10 ** k < 1 or m // 10 ** k > 9 or m % 10 ** k:
                    continue
                j, nb = m // 10 ** k, n // m
                b = s[:nb * j].reshape(nb, j)
                eb = E[:nb * j].reshape(nb, j).sum(1)
                d = b[1:].sum(1) - b[:-1].sum(1)
                ot = o[np.arange(1, nb) * j][:, None]        # the tile of the term's second bin
                a = np.abs(b[1:] - ot).sum(1) + np.abs(b[:-1] - ot).sum(1)
                ed = (eb[1:] + eb[:-1] + _g(j + 1) * (a + np.abs(d))) * (1 + 4 * U)
                et = ed * (2 * np.abs(d) + ed)
                D = max(30 + 5 + 16 + -(-chunks // 32) + 5, -(-nb // 512) + 5 + 16 + 2)
                c = 0.5 / ((nb - 1) * float(m) * m)
                out[i] = (c * ((1 + _g(D)) * et.sum() + _g(D) * exact[i] / c) + _g(4) * exact[i]) * (1 + 1e-6)
            if L < 10 or not any(m // 10 ** (k + 1) >= 1 for m in mult):
                break
            nl = L // 10
            ch = s[:nl * 10].reshape(nl, 10)
            od = o[:nl * 10:10][:, None] if not rest else 0.0
            s1 = ch.sum(1)
            E = (E[:nl * 10].reshape(nl, 10).sum(1) +
                 _g(11) * (np.abs(ch - od).sum(1) + 10 * np.abs(od).ravel() + np.abs(s1))) * (1 + 4 * U)
            s = s1
    return out


# ---------------------------------------------------------------------------------------------------------
# the front ends
# ---------------------------------------------------------------------------------------------------------
def _run(eng, fs, x, how):
    """x: [S, n] -> avar [S, ntau] through the front end `how`, and tau."""
    S, n = x.shape
    if how == 'stream':              # contiguous: allan_stream_kernel if the rows are 16-byte aligned (n even)
        av, tau = eng.allan(fs, eng.to_device(x), n, S)
    elif how == 'full_misaligned':   # x[:, 1:] of a contiguous buffer: allan_full_kernel<true>
        buf = np.zeros((S, n + 2))
        buf[:, 1:n + 1] = x
        t = eng.to_device(buf)
        av, tau = eng.allan(fs, t.view(-1)[1:], n, S, outer_stride=n + 2)
    elif how == 'full_odd_stride':   # aligned base, odd row stride: allan_full_kernel<true>
        p = n + 1 + (n % 2)
        buf = np.zeros((S + 1, p))
        buf[:S, :n] = x
        av, tau = eng.allan(fs, eng.to_device(buf), n, S, outer_stride=p)
    elif how == 'full_triads':       # interleaved triads: allan_full_kernel<false>
        R = -(-S // 3)
        buf = np.zeros((R, n, 3))
        for s in range(S):
            buf[s // 3, :, s % 3] = x[s]
        av, tau = eng.allan(fs, eng.to_device(buf), n, 3 * R, inner=3, outer_stride=3 * n, sample_stride=3)
        av = av[:S]
    else:
        raise ValueError(how)
    torch.cuda.synchronize()
    return av.cpu().numpy(), tau.cpu().numpy()


FRONT_ENDS = ('stream', 'full_misaligned', 'full_odd_stride', 'full_triads')


def _path_name(how, n):
    if n <= CH:
        return 'rest'
    return 'full_odd_stride' if how == 'stream' and n % 2 else how


def _check(got, x, fs, exact, what, how, bound=None):
    """got [ntau] of series x against its exact reference (avar, tau): the class, then the bound."""
    ex, _ = exact
    assert got.shape == ex.shape, what
    assert np.array_equal(np.isnan(got), np.isnan(ex)), (what, got, ex)
    assert np.array_equal(np.isinf(got), np.isinf(ex)), (what, got, ex)
    assert not (got < 0).any(), what
    fin = np.isfinite(ex)
    if not fin.any():
        return
    b = k4_bound(x, fs, np.where(fin, ex, 0.0)) if bound is None else bound
    err = np.abs(got[fin] - ex[fin])
    assert (err <= b[fin]).all(), (what, np.nonzero(err > b[fin]), (err / b[fin]).max())
    r = float(np.max(err / b[fin], initial=0.0, where=b[fin] > 0))
    key = _path_name(how, len(x))
    WORST[key] = max(WORST.get(key, 0.0), r)


def _batch_check(eng, fs, xs, hows=FRONT_ENDS, exacts=None, what=''):
    xs = np.atleast_2d(np.asarray(xs, dtype=np.float64))
    exacts = exacts or [ae.allan_var(x, fs) for x in xs]
    with np.errstate(invalid='ignore', over='ignore'):
        bounds = [k4_bound(x, fs, np.where(np.isfinite(e[0]), e[0], 0.0)) for x, e in zip(xs, exacts)]
    for how in hows:
        av, tau = _run(eng, fs, xs, how)
        for s in range(xs.shape[0]):
            assert np.array_equal(tau, exacts[s][1]), (what, how)
            _check(av[s], xs[s], fs, exacts[s], '%s %s series %d' % (what, how, s), how, bounds[s])
    return exacts


# ---------------------------------------------------------------------------------------------------------
# shapes: every path, ragged last chunks at levels 0, 1, 2, the tile count against the SM count
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [81, 4000, 5040, 5041, 50400, 50409, 50410, 50419, 503999, 504001])
def test_every_path_at_the_level_handoffs(eng, n):
    rng = np.random.default_rng(n)
    x = np.stack([0.3 * rng.standard_normal(n) + 2.0, np.cumsum(rng.standard_normal(n)) * 1e-3])
    _batch_check(eng, 1.0 if n > 100 else 9.0, x, what='n=%d' % n)


@pytest.mark.parametrize('level', [0, 1, 2])
def test_ragged_last_chunk_sizes(eng, level):
    """The last chunk of level `level` holds r = 1, 9, 10, 11 and 5039 elements (a full chunk before it)."""
    rows = []
    for r in (1, 9, 10, 11, 5039):
        n = (CH + r) * 10 ** level + 7 * (level > 0)
        rows.append(n)
    for n in rows:
        x = np.random.default_rng(n).standard_normal(n) * 0.1 + 1.0
        _batch_check(eng, 1.0, x[None], hows=('stream', 'full_triads') if level == 2 else FRONT_ENDS,
                     what='level %d n=%d' % (level, n))


def test_inner_two_with_unit_stride(eng):
    """inner = 2, sample_stride = 1: series 2q + 1 starts one element after series 2q (allan_full_kernel<true>)."""
    n = 50411
    buf = np.random.default_rng(2).standard_normal((2, n + 3)) + 5.0
    av, tau = eng.allan(1.0, eng.to_device(buf), n, 4, inner=2, outer_stride=n + 3)
    av = av.cpu().numpy()
    for s in range(4):
        x = buf[s // 2, s % 2:s % 2 + n]
        _check(av[s], x, 1.0, ae.allan_var(x, 1.0), 'inner=2 series %d' % s, 'full_inner2')


def test_tiles_against_the_sm_count(eng, sms):
    """Stream kernel with tiles = sms - 1, sms, sms + 1 and 3 sms + 1 of one contiguous series (more chunks than
    the grid: advance() with step_s = 0), and a batch of more two-chunk series than half the grid."""
    for tiles in (sms - 1, sms, sms + 1, 3 * sms + 1):
        n = (tiles - 1) * CH + 2520          # even: 16-byte aligned rows
        x = np.random.default_rng(tiles).standard_normal(n) * 1e-2 + 9.8
        _batch_check(eng, 100.0, x[None], hows=('stream',), what='tiles=%d' % tiles)
    S = (sms + 1) // 2 + 1
    x = np.random.default_rng(5).standard_normal((S, 5040 + 2520))
    _batch_check(eng, 1.0, x, hows=('stream',), what='%d series' % S)
    # bit-identical whatever the batch: alone, first, last, and on every front end
    av, _ = _run(eng, 1.0, x, 'stream')
    for s in (0, S - 1):
        a1, _ = _run(eng, 1.0, x[s:s + 1], 'stream')
        assert np.array_equal(a1[0], av[s])
    a2, _ = _run(eng, 1.0, np.concatenate([x[3:], x[:3]]), 'stream')
    assert np.array_equal(a2[-3:], av[:3]) and np.array_equal(a2[:-3], av[3:])


# ---------------------------------------------------------------------------------------------------------
# the tau grid
# ---------------------------------------------------------------------------------------------------------
def test_tau_grid_edges(eng):
    # max_bin = 1000 exactly for n = 9000..9008 (the reference drops m = 1000: ceil(log10(1000)) = 3), 9009 keeps it
    for n in list(range(9000, 9009)) + [9009]:
        x = np.random.default_rng(n).standard_normal(n)
        av, tau = _run(eng, 1.0, x[None], 'stream')
        ex = ae.allan_var(x, 1.0)
        assert np.array_equal(tau, ex[1]) and (1000 in onp.allan_multipliers(n, 1.0)) == (n == 9009)
        _check(av[0], x, 1.0, ex, 'n=%d' % n, 'stream')
    # a top level with jmax = 1, 2, 9
    for n, jmax in ((90009, 1), (180000, 2), (810000, 9)):
        mult = onp.allan_multipliers(n, 1.0)
        assert mult[-1] == jmax * 10000
        x = np.random.default_rng(jmax).standard_normal(n)
        _batch_check(eng, 1.0, x[None], hows=('stream', 'full_triads'), what='jmax=%d' % jmax)
    # non-integer rates: tau = m * (1 / fs) bit for bit
    for fs in (3.7, 100.0 / 3.0, 0.9):
        x = np.random.default_rng(1).standard_normal(60001)
        _batch_check(eng, fs, x[None], hows=('stream', 'full_misaligned'), what='fs=%r' % fs)
    # max_bin * ts exactly 1, and just below (no tau at all)
    assert 100 * (1.0 / 100.0) == 1.0
    av, tau = _run(eng, 100.0, np.ones((1, 900)), 'stream')
    assert np.array_equal(tau, ae.allan_var(np.ones(900), 100.0)[1]) and len(tau) == 18 and np.all(av == 0.0)
    av, tau = _run(eng, 100.0, np.ones((1, 899)), 'stream')
    assert av.shape == (1, 0) and tau.shape == (0,)


# ---------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------
def test_offsets_ramps_and_random_walks(eng):
    n = 560018
    rng = np.random.default_rng(17)
    w = rng.standard_normal((4, n))
    x = np.stack([1e4 + w[0], 1e7 + w[1], 5.0 + 1e-4 * np.arange(n) + w[2], np.cumsum(w[3])])
    _batch_check(eng, 100.0, x, what='offsets/ramp/walk')


@pytest.mark.parametrize('n', [4000, 50410, 560017])
def test_periodic_series_give_exactly_zero_where_the_period_divides_m(eng, n):
    """Period p: every level-0 cluster of m = p, 2p, .. samples holds the same values in the same order, so
    adjacent clusters summed by the same operation tree give exactly 0 (also across item and tile edges)."""
    rng = np.random.default_rng(4)
    for p in range(2, 10):
        # 24 periods each: a changed summation order rounds differently for only some of them
        x = np.stack([np.tile(rng.standard_normal(p) + c, -(-n // p))[:n] for c in (0.0, 1e4) * 12])
        for how in FRONT_ENDS:
            av, _ = _run(eng, 1.0, x, how)
            for m in range(p, 10, p):
                assert np.all(av[:, m - 1] == 0.0), (p, m, how, av[:, m - 1])


@pytest.mark.parametrize('n', [4000, 50410, 560017])
def test_constant_series_is_exactly_zero(eng, n):
    """Adjacent clusters are summed by the same operation tree on every path: exactly 0 at every tau."""
    x = np.stack([np.full(n, 0.1), np.full(n, 1.0 / 3.0), np.full(n, -9.80665)])
    for how in FRONT_ENDS:
        av, _ = _run(eng, 1.0, x, how)
        assert av.size > 0 and np.all(av == 0.0), (how, np.nonzero(av))


# ---------------------------------------------------------------------------------------------------------
# non-finite samples
# ---------------------------------------------------------------------------------------------------------
def _spots(n):
    """Positions: x[0]; a chunk's halo start at level 0 and as the first decade of a tile at levels 1 and 2;
    inside the ragged last chunk; the last sample; the tail past nb * m of the longest tau."""
    p = [0, CH - 9, 10 * (CH - 9), 100 * (CH - 9), (n // CH) * CH + 3, n - 1]
    top = onp.allan_multipliers(n, 1.0)[-1]
    p.append((n // top) * top + 1)
    return [q for q in p if q < n]


KINDS = {'nan': [(0, np.nan)], '+inf': [(0, np.inf)], '-inf': [(0, -np.inf)],
         'both': [(0, np.inf), (1, -np.inf)]}


@pytest.mark.parametrize('n', [4000, 50419, 560017])
def test_non_finite_samples_on_every_path(eng, n):
    rng = np.random.default_rng(n + 1)
    base = rng.standard_normal(n) * 0.2 + 3.0
    fin_exact = ae.allan_var(base, 1.0)
    rows, exacts = [], []
    mult = onp.allan_multipliers(n, 1.0)
    for p in _spots(n):
        for kind, spots in KINDS.items():
            x = base.copy()
            for dq, v in spots:
                if p + dq < n:
                    x[p + dq] = v
            cls = ae.nonfinite_class(x, mult)
            ex = fin_exact[0].copy()            # finite taus do not see the samples that changed
            ex[cls == 1] = np.inf
            ex[cls == 2] = np.nan
            rows.append(x)
            exacts.append((ex, fin_exact[1]))
    # two +inf in adjacent bins of m = 1 (NaN there), two in one bin of m = 2 (+inf there)
    x = base.copy()
    x[n // 2 - (n // 2) % 2] = x[n // 2 - (n // 2) % 2 + 1] = np.inf
    rows.append(x)
    exacts.append(ae.allan_var(x, 1.0))
    assert np.isnan(exacts[-1][0][0]) and exacts[-1][0][1] == np.inf
    _batch_check(eng, 1.0, np.stack(rows), exacts=exacts, what='non-finite n=%d' % n)
    if n == 4000:
        # x[0] = +inf and n <= 5040: +inf at every tau
        x = base.copy()
        x[0] = np.inf
        av, _ = _run(eng, 1.0, x[None], 'stream')
        assert np.all(av == np.inf)


# ---------------------------------------------------------------------------------------------------------
# the generating front end (K1 fused into level 0)
# ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [5041, 10080, 10081, 50410])
def test_gen_kernel_walks_several_series(eng, sms, n):
    """R = 50 runs, 300 series on `sms` CTAs: every CTA walks two or three series.  Against K1 -> K4 on the
    materialised series; run r of the R = 50 launch bit-identical to the same run launched alone."""
    from gnss_ins_sim_b200 import imu_model
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    rng = np.random.default_rng(n)
    ref_gyro = eng.to_device(0.01 * rng.standard_normal((n, 3)))
    ref_accel = eng.to_device(np.array([0.3, -0.2, -9.8]) + 0.01 * rng.standard_normal((n, 3)))
    R, r0, seed = 50, 11, 7
    assert 6 * R > 2 * sms
    avar, tau = eng.allan_mc(200.0, R, ref_gyro, ref_accel, imu.gyro_err, imu.accel_err, seed, run_offset=r0)
    gyro, accel = eng.imu_noise(200.0, R, ref_gyro, ref_accel, imu.gyro_err, imu.accel_err, seed,
                                run_offset=r0, layout=eng.LAYOUT_CHANNEL_MAJOR)
    av_a, _ = eng.allan(200.0, accel, n, R * 3)
    av_g, _ = eng.allan(200.0, gyro, n, R * 3)
    ref = np.concatenate([av_a.cpu().numpy().reshape(R, 3, -1), av_g.cpu().numpy().reshape(R, 3, -1)], axis=1)
    got = avar.cpu().numpy()
    assert got.shape == ref.shape and np.all(ref > 0)
    assert np.abs(got / ref - 1.0).max() < 1e-9
    for r in (0, 22, 44, 49):       # first in its CTA, then second and third (series 6r + c on CTA (6r + c) % sms)
        a1, _ = eng.allan_mc(200.0, 1, ref_gyro, ref_accel, imu.gyro_err, imu.accel_err, seed, run_offset=r0 + r)
        assert np.array_equal(a1.cpu().numpy()[0], got[r]), r
    # the series of one run, held to the exact reference
    x = np.concatenate([accel[7].cpu().numpy(), gyro[7].cpu().numpy()])
    for c in range(6):
        _check(got[7, c], x[c], 200.0, ae.allan_var(x[c], 200.0), 'gen run 7 ch %d' % c, 'gen')


# ---------------------------------------------------------------------------------------------------------
# the plugin and the logged-data directory
# ---------------------------------------------------------------------------------------------------------
def test_plugin_with_nan_and_inf(eng):
    from gnss_ins_sim_b200.allan_analysis import Allan
    R, n, fs = 2, 20011, 50.0
    rng = np.random.default_rng(9)
    acm = rng.standard_normal((R, 3, n)) * 0.02 + np.array([0.1, -0.2, -9.8])[None, :, None]
    gcm = rng.standard_normal((R, 3, n)) * 1e-3
    acm[0, 1, 777] = np.nan
    acm[1, 2, 12000] = np.inf
    gcm[1, 0, 0] = -np.inf
    tau, a1, g1 = Allan().run_batch(fs, acm, gcm, channel_major=True)
    _, a2, g2 = Allan().run_batch(fs, acm.transpose(0, 2, 1), gcm.transpose(0, 2, 1))
    assert np.array_equal(a1, a2, equal_nan=True) and np.array_equal(g1, g2, equal_nan=True)
    for r in range(R):
        for c in range(3):
            for got, x in ((a1[r, :, c], acm[r, c]), (g1[r, :, c], gcm[r, c])):
                ex, et = ae.allan_var(x, fs)
                assert np.array_equal(tau, et)
                assert np.array_equal(np.isnan(got), np.isnan(ex)) and np.array_equal(np.isinf(got), np.isinf(ex))
                f = np.isfinite(ex)
                assert np.allclose(got[f] ** 2, ex[f], rtol=1e-9, atol=0.0), (r, c)
    assert np.isnan(a1[0, 0, 1]) and np.isinf(a1[1, -1, 2]) and np.isinf(g1[1, 0, 0])


def test_logged_directory_with_a_nan_gap_and_an_inf(eng, tmp_path):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    g = load_golden('logged_bosch.npz')
    g['gyro'] = g['gyro'].copy()
    g['accel'] = g['accel'].copy()
    g['gyro'][400:410, 1] = np.nan
    g['accel'][777, 0] = np.inf
    d = write_logged_dir(str(tmp_path / 'bosch'), g, deg=False)
    sim = Sim([100.0, 0.0, 0.0], d, ref_frame=0, imu=None, algorithm=Allan())
    sim.run(1)
    ada, adg, tau = (sim.get_data([k])[0]['algo0_0'] for k in ('ad_accel', 'ad_gyro', 'algo_time'))
    for ad, x in ((ada, g['accel']), (adg, g['gyro'])):
        for c in range(3):
            ex, et = ae.allan_var(x[:, c], 100.0)
            assert np.array_equal(tau, et)
            assert np.array_equal(np.isnan(ad[:, c]), np.isnan(ex)) and np.array_equal(np.isinf(ad[:, c]), np.isinf(ex))
            f = np.isfinite(ex)
            assert np.allclose(ad[f, c] ** 2, ex[f], rtol=1e-9, atol=0.0)
    assert np.isnan(adg[:, 1]).any() and np.isinf(ada[:, 0]).any() and np.isfinite(ada[:, 1]).all()
