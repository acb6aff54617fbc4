"""K4o, the overlapping Allan variance and its Hadamard form, held to the exact reference (oracle/oallan_exact.py)
on every front end of oallan_launch, at its tile and grid edges, with non-finite samples across tiles and at the
ends of the float64 range.

Error bound (oallan_exact.k4o_bound).  u = 2^-53, g_p = p u / (1 - p u).  For a tau m with K terms (K = n - 2m + 1,
Allan; n - 3m + 1, Hadamard), K4o's own order of operations gives:
  * the shift: y_i = fl(x_i - x_0) is NOT error-free (an outlier x_0, or a drift wider than 53 bits of the
    samples' grid, rounds it).  Its error delta_i is computed exactly (TwoSum) and enters a term through its
    windows: sum_A |delta| + sum_B |delta| (Allan), sum_S0 + 2 sum_S1 + sum_S2 (Hadamard);
  * the double-double prefix: a sample reaches C[i] through <= 9 thread-serial dd_add_d, 8 Hillis-Steele steps,
    the exclusive combine and the carry add of its tile, or, from an earlier tile, its tile total (9 + 8) and
    <= tiles serial carry adds: <= tile(i) + 20 adds in all.  Each double-double add errs by <= 8 u^2 (|a| + |b|),
    so |C^[i] - C_y[i]| <= eps_i = 8 u^2 (tile(i) + 20) sum_{q<i} |y_q|.  A term takes eps with the weights of
    its prefix points: 1, 2, 1 (Allan), 1, 3, 3, 1 (Hadamard);
  * the term.  Allan: D_m, D_2m by dd_diff (exact TwoDiff of the hi parts, then two lo adds), then
    t = (D_2m.hi - 2 D_m.hi) + (D_2m.lo - 2 D_m.lo), three roundings: |t^ - t| <= 2 u |t| + 5 u Lambda, with
    Lambda = u (|D_2m| + 2 |D_m|) + u (3 |C_k| + 2 |C_k+m| + |C_k+2m|) bounding the lo parts.  Hadamard: the three
    window sums by dd_diff, then the hi subtractions S2.hi - S1.hi and S1.hi - S0.hi, each exact when its operands
    are within a factor of two (Sterbenz) and otherwise off by u |S2 - S1| or u |S1 - S0|, their difference and the
    final add (2 u |t|), and the lo sums (6 u Lambda_H, Lambda_H = u (|S0| + 2|S1| + |S2|) + u (|C_k| + 3|C_k+m| +
    3|C_k+2m| + |C_k+3m|));
  * the square by FMA: |t^^2 - t^2| <= e (2 |t| + e) for a term error e, its rounding folded into the sum;
  * the folds: a chain of <= 8 FMAs in a thread, a 5-step butterfly, 8 warps in order, then ceil(sq_tiles / 32)
    lane adds and a 5-step butterfly in pass 5: depth D = 26 + ceil(sq_tiles / 32), all terms >= 0, g_D of the sum;
  * the normaliser: 2.0 * m * m * M (6.0 * m * m * H) rounds once it passes 2^53 (config-4 lengths), and the
    division rounds once: g_3;
  * gradual underflow: the FMA squares and the division, each off by at most 2^-1075 absolute in the subnormal
    range: 2^-1074 (1 + 2 K / den).
|K4o - exact| <= bound is asserted at every finite tau.  A NaN or +inf must be of the exact reference's class;
a series of finite samples never gives NaN, and gives +inf at a finite exact tau only where the float64 sum of the
squared terms passes DBL_MAX (1e160 samples).  Integer data with |C|, sum t^2 and the normaliser below 2^53 make
every K4o operation exact: there K4o equals the exact reference bit for bit."""
import numpy as np
import pytest

import oallan_exact as ox
from conftest import load_golden, write_logged_dir

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

SCAN, SQ = 2304, 2048
DBL_MAX = np.finfo(np.float64).max
WORST = {}          # (form, front end) -> worst |K4o - exact| / bound, printed at the end of the module
FORMS = {'allan': False, 'hadamard': True}


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nK4o worst |K4o - exact| / bound per form and front end: ' +
          ', '.join('%s/%s %.3g' % (f, h, r) for (f, h), r in sorted(WORST.items())))


# ---------------------------------------------------------------------------------------------------------------
# the front ends
# ---------------------------------------------------------------------------------------------------------------
def _run(eng, fs, x, had, how='rows'):
    """x: [S, n] -> var [S, ntau] through the front end `how`, and tau."""
    fn = eng.ohadamard if had else eng.oallan
    S, n = x.shape
    if how == 'rows':
        v, tau = fn(fs, eng.to_device(x), n, S)
    elif how == 'misaligned':                    # x[:, 1:] of a contiguous buffer: an 8-byte-aligned base
        buf = np.zeros((S, n + 2))
        buf[:, 1:n + 1] = x
        v, tau = fn(fs, eng.to_device(buf).view(-1)[1:], n, S, outer_stride=n + 2)
    elif how == 'odd_stride':
        p = n + 1 + (n % 2)
        buf = np.zeros((S + 1, p))
        buf[:S, :n] = x
        v, tau = fn(fs, eng.to_device(buf), n, S, outer_stride=p)
    elif how in ('inner2', 'triads', 'inner6'):  # [R, n, inner], series s = channel s % inner of record s // inner
        inner = {'inner2': 2, 'triads': 3, 'inner6': 6}[how]
        R = -(-S // inner)
        buf = np.zeros((R, n, inner))
        for s in range(S):
            buf[s // inner, :, s % inner] = x[s]
        v, tau = fn(fs, eng.to_device(buf), n, inner * R, inner=inner, outer_stride=inner * n, sample_stride=inner)
        v = v[:S]
    elif how == 'stride5':                       # every fifth sample of a row
        buf = np.zeros((S, 5 * n))
        buf[:, ::5] = x
        v, tau = fn(fs, eng.to_device(buf), n, S, outer_stride=5 * n, sample_stride=5)
    else:
        raise ValueError(how)
    torch.cuda.synchronize()
    return v.cpu().numpy(), tau.cpu().numpy()


FRONT_ENDS = ('rows', 'misaligned', 'odd_stride', 'inner2', 'triads', 'inner6', 'stride5')


def _reference(x, fs, had, mult=None):
    """(exact, tau, info, bound); the bound only for series of finite samples."""
    if np.isfinite(x).all():
        return ox.k4o_bound(x, fs, had, mult)
    ex, tau, info = ox.exact(x, fs, had, mult)
    return ex, tau, info, None


def _check(got, x, ref, what, key, cols=None):
    """got [ntau] (or its columns cols of the full grid) of series x against (exact, tau, info, bound)."""
    ex, _, info, bound = ref
    if cols is not None:
        got = got[cols]
    assert got.shape == ex.shape, what
    cls = info['cls']
    assert np.array_equal(np.isnan(got), cls == 2), (what, got, cls)
    assert np.all(got[cls == 1] == np.inf), (what, got, cls)
    fin = cls == 0
    if np.isfinite(x).all():
        assert not np.isnan(got).any(), (what, 'a series of finite samples gave NaN', got)
    assert not (got < 0).any(), what
    # an overflowing exact ratio is +inf; K4o may also overflow where its float64 sum of squares cannot hold
    inf_ok = fin & ((ex == np.inf) | (info['st2'] > DBL_MAX / (1.0 + 1e-12)))
    assert np.all(got[fin & (ex == np.inf)] == np.inf), (what, got, ex)
    chk = fin & ~inf_ok
    assert np.all(np.isfinite(got[chk])), (what, got, ex)
    if not chk.any():
        return
    err = np.abs(got[chk] - ex[chk])
    b = bound[chk]
    assert np.all(err <= b), (what, np.nonzero(err > b), (err / b).max(), got[chk], ex[chk])
    WORST[key] = max(WORST.get(key, 0.0), float((err / b).max()))


def _batch(eng, fs, xs, hows=('rows',), forms=FORMS, what='', refs=None):
    xs = np.atleast_2d(np.asarray(xs, dtype=np.float64))
    out = {}
    for form, had in forms.items():
        rs = refs[form] if refs else [_reference(x, fs, had) for x in xs]
        for how in hows:
            v, tau = _run(eng, fs, xs, had, how)
            for s in range(xs.shape[0]):
                assert np.array_equal(tau, rs[s][1]), (what, how)
                _check(v[s], xs[s], rs[s], '%s %s %s series %d' % (what, form, how, s), (form, how))
        out[form] = rs
    return out


# ---------------------------------------------------------------------------------------------------------------
# the edges: scan tiles (2304), output tiles (2048) and the grid (m = floor(n / 9))
# ---------------------------------------------------------------------------------------------------------------
def _edge_lengths():
    ns = {9, 8, 2304 * 5 - 1, 2304 * 5, 2304 * 5 + 1}
    for m in (1, 10, 90, 900):
        ns |= {9 * m, 9 * m - 1}
    for m, t in ((1, 3), (10, 4), (100, 6)):          # the last offset n - 2m (n - 3m) at 2048 t - 1, 2048 t, + 1
        for span in (2, 3):
            ns |= {SQ * t + span * m + d for d in (-1, 0, 1)}
    return sorted(ns)


EDGES = _edge_lengths()


def _integer_rows(n, rng):
    """Small integers, integers times 2^-7 on an offset (quantised sensor counts), a +-1 walk: every K4o operation
    on them is exact."""
    a = rng.integers(-8, 9, n).astype(np.float64)
    b = (4096.0 + rng.integers(-20, 21, n)) * 2.0 ** -7
    c = np.cumsum(rng.integers(-1, 2, n)).astype(np.float64)
    return np.stack([a, b, c])


@pytest.mark.parametrize('n', EDGES)
def test_integer_data_bit_for_bit(eng, n):
    x = _integer_rows(n, np.random.default_rng(n))
    for form, had in FORMS.items():
        for how in ('rows', 'triads'):
            v, tau = _run(eng, 1.0, x, had, how)
            for s in range(3):
                ex, et, info = ox.exact(x[s], 1.0, had)
                assert np.array_equal(tau, et) and v.shape[1] == len(ex), (n, form)
                assert np.array_equal(v[s], ex), (n, form, how, s, v[s], ex)
    if n == 8:
        assert v.shape == (3, 0)


def _kinds(n, rng):
    i = np.arange(n, dtype=np.float64)
    w = rng.standard_normal((7, n))
    x0 = w[5].copy()
    x0[0] = 3e3
    # drift: a rate ramp from an exact 0 with full-mantissa samples, so that only the double-double prefix keeps
    # the sums of a thread's nine samples (an uncompensated thread run shows in the Hadamard terms)
    return {'offset_1e4': 1e4 + w[0], 'offset_1e7': 1e7 + w[1],
            'drift': np.where(i == 0, 0.0, 1e-3 * i + 1e-6 * w[6]),
            'ramp': 1e4 + 1e-3 * i + 1e-3 * w[2], 'quadratic': 1.0 + 1e-3 * i + 2e-7 * i * i + 0.01 * w[3],
            'walk': np.cumsum(w[4]), 'outlier_x0': x0}


@pytest.mark.parametrize('n', [2304 * 5 - 1, 2304 * 5 + 1, SQ * 3 + 2, SQ * 3 + 3, 8099, 8100, 810 * 9 + 17])
def test_finite_series_where_rounding_matters_at_the_edges(eng, n):
    k = _kinds(n, np.random.default_rng(n))
    _batch(eng, 1.0, np.stack(list(k.values())), hows=('rows', 'odd_stride'), what='n=%d' % n)


@pytest.mark.parametrize('kind', ['offset_1e4', 'offset_1e7', 'drift', 'ramp', 'quadratic', 'walk', 'outlier_x0'])
def test_a_million_samples(eng, kind):
    n = 10 ** 6
    x = _kinds(n, np.random.default_rng(61))[kind]
    _batch(eng, 100.0, x[None], what=kind)


def test_config4_length_channel_at_a_handful_of_tau(eng):
    """One accelerometer z channel at BASELINE config-4 length (14.4 M samples @400 Hz), K1's own draw: the exact
    reference at five taus of the 55 (both normalisers pass 2^53 at the longest)."""
    from gnss_ins_sim_b200 import imu_model
    n, fs = 14400000, 400.0
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    ref_gyro = eng.to_device(np.zeros((n, 3)))
    ref_accel = eng.to_device(np.tile([0.0, 0.0, -9.8], (n, 1)))
    _, accel = eng.imu_noise(fs, 1, ref_gyro, ref_accel, imu.gyro_err, imu.accel_err, 5,
                             layout=eng.LAYOUT_CHANNEL_MAJOR)
    z = accel[0, 2:3].contiguous()
    del ref_gyro, ref_accel
    grid = ox._grid(n, fs)[0]
    pick = [1, 7, 1000, 90000, 1000000]
    cols = [grid.index(m) for m in pick]
    assert 2.0 * 1e6 * 1e6 * (n - 2e6 + 1) > 2.0 ** 53
    zz = z.cpu().numpy()[0]
    for form, had in FORMS.items():
        fn = eng.ohadamard if had else eng.oallan
        v, tau = fn(fs, z, n, 1)
        v = v.cpu().numpy()[0]
        ref = ox.k4o_bound(zz, fs, had, pick)
        assert np.array_equal(tau.cpu().numpy()[cols], ref[1])
        _check(v, zz, ref, 'config-4 accel z %s' % form, (form, 'config4'), cols=cols)


# ---------------------------------------------------------------------------------------------------------------
# non-finite samples across tiles
# ---------------------------------------------------------------------------------------------------------------
def test_non_finite_samples_across_tiles(eng):
    n = 70001                                       # 31 scan tiles, m up to 7000: windows wider than 3 tiles
    rng = np.random.default_rng(8)
    base = rng.standard_normal(n) * 0.3 + 2.0
    spots = [[(n - 5, np.nan)],                                         # only in the last, ragged tile
             [(SCAN - 1, np.inf), (4 * SCAN, -np.inf)],                 # tile 0 and tile 4
             [(0, np.inf)], [(0, -np.inf)],
             [(3 * SCAN - 1, np.inf)], [(3 * SCAN, -np.inf)], [(n - 1, np.inf)],
             [(5000, np.inf), (5003, np.inf), (5100, np.inf), (5050, -np.inf), (20000, -np.inf), (20001, -np.inf)],
             [(7000, np.nan), (30000, np.inf)], [(12, -np.inf), (60000, np.nan)]]
    rows = [base]
    for sp in spots:
        x = base.copy()
        for i, val in sp:
            x[i] = val
        rows.append(x)
    rows.append(1e4 + 1e-3 * np.arange(n) + 1e-3 * rng.standard_normal(n))
    xs = np.stack(rows)
    out = _batch(eng, 1.0, xs, hows=('rows', 'triads'), what='non-finite')
    for form in FORMS:                              # the tile-0 / tile-4 pair: NaN at some taus, +inf at others
        cls = out[form][2][2]['cls']
        assert (cls == 2).any() and (cls == 1).any(), (form, cls)
        assert np.all(out[form][3][2]['cls'] == 1)  # x[0] = +inf: +inf everywhere


# ---------------------------------------------------------------------------------------------------------------
# magnitude
# ---------------------------------------------------------------------------------------------------------------
def test_tiny_and_huge_magnitudes(eng):
    rng = np.random.default_rng(150)
    n = 5 * SCAN + 3
    w = rng.standard_normal((4, n))
    xs = np.stack([1e-150 * w[0], 1e-157 * w[1], 1e150 * w[2], 1e160 * w[3]])
    out = _batch(eng, 1.0, xs, hows=('rows', 'misaligned'), what='magnitude')
    ex157 = out['allan'][1][0]
    assert (ex157 < 2.2250738585072014e-308).any()          # the 1e-157 series reaches gradual underflow
    v, _ = _run(eng, 1.0, xs[3:], False)
    assert np.all(v == np.inf)                              # every square past DBL_MAX


def test_overflowing_prefix_gives_inf_not_nan(eng):
    """x_0 = -1e305, the rest +1e305: x - x_0 = 2e305 is finite, the prefix overflows within the first tile, and
    two_sum of an infinite sum is NaN.  The exact value is +inf at every tau, and that is what K4o reports."""
    xs = []
    for n in (2 * SCAN + 5, 9 * SCAN):
        x = np.full(n, 1e305)
        x[0] = -1e305
        xs.append(x)
    for x in xs:
        for form, had in FORMS.items():
            v, _ = _run(eng, 1.0, x[None], had)
            ex, _, info = ox.exact(x, 1.0, had)
            assert np.all(ex == np.inf) and np.all(info['cls'] == 0)
            assert np.all(v[0] == np.inf), (form, len(x), v)


# ---------------------------------------------------------------------------------------------------------------
# front ends
# ---------------------------------------------------------------------------------------------------------------
def test_every_front_end(eng):
    n = 3 * SCAN + 11
    rng = np.random.default_rng(12)
    k = _kinds(n, rng)
    xs = np.stack(list(k.values()) + [rng.standard_normal(n)])
    _batch(eng, 20.0, xs, hows=FRONT_ENDS, what='front ends')


def test_a_batch_of_3000_short_series_is_each_series_alone(eng):
    n = 200
    rng = np.random.default_rng(3000)
    xs = rng.standard_normal((3000, n)) * rng.uniform(0.1, 10.0, (3000, 1)) + rng.uniform(-1e3, 1e3, (3000, 1))
    for form, had in FORMS.items():
        fn = eng.ohadamard if had else eng.oallan
        dx = eng.to_device(xs)
        batch, _ = fn(10.0, dx, n, 3000)
        alone = torch.stack([fn(10.0, dx[s:s + 1], n, 1)[0][0] for s in range(3000)])
        assert torch.equal(batch, alone), form
        batch = batch.cpu().numpy()
        for s in (0, 1, 1499, 2999):
            _check(batch[s], xs[s], _reference(xs[s], 10.0, had), '3000 %s %d' % (form, s), (form, 'batch3000'))


def test_plugins_on_both_layouts(eng):
    """Allan(overlapping=True) and Hadamard() run_batch: the deviation is sqrt of the variance K4o gives the same
    series alone, on the channel-major and the interleaved layout; the variances are held to the exact reference."""
    from gnss_ins_sim_b200.allan_analysis import Allan, Hadamard
    R, n, fs = 2, 3 * SCAN + 100, 50.0
    rng = np.random.default_rng(77)
    acm = rng.standard_normal((R, 3, n)) * 0.02 + np.array([0.1, -0.2, -9.8])[None, :, None]
    gcm = rng.standard_normal((R, 3, n)) * 1e-3 + 1e-5 * np.arange(n)
    for plugin, had in ((Allan(overlapping=True), False), (Hadamard(), True)):
        tau, a1, g1 = plugin.run_batch(fs, acm, gcm, channel_major=True)
        _, a2, g2 = plugin.run_batch(fs, acm.transpose(0, 2, 1), gcm.transpose(0, 2, 1))
        assert np.array_equal(a1, a2) and np.array_equal(g1, g2)
        for dev, data, what in ((a1, acm, 'accel'), (g1, gcm, 'gyro')):
            var, t = _run(eng, fs, data.reshape(R * 3, n), had)
            assert np.array_equal(t, tau)
            assert np.array_equal(dev.transpose(0, 2, 1).reshape(R * 3, -1), np.sqrt(var)), what
            for s in (0, 5):
                _check(var[s], data.reshape(R * 3, n)[s], _reference(data.reshape(R * 3, n)[s], fs, had),
                       'plugin %s %s %d' % (type(plugin).__name__, what, s), ('allan' if not had else 'hadamard',
                                                                           'plugin'))


@pytest.mark.parametrize('plugin', ['Allan', 'Hadamard'])
def test_logged_directory_with_inf_and_nan_channels(eng, tmp_path, plugin):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200 import allan_analysis
    g = load_golden('logged_bosch.npz')
    n = 7 * 1000 + 13
    rng = np.random.default_rng(5)
    gyro = np.tile(g['gyro'], (8, 1))[:n] + 1e-4 * rng.standard_normal((n, 3))
    accel = np.tile(g['accel'], (8, 1))[:n] + 1e-3 * rng.standard_normal((n, 3))
    gyro[2 * SCAN + 100, 1] = np.inf                     # scan tile 2 of gyro y
    accel[1500, 2] = np.nan
    d = write_logged_dir(str(tmp_path / 'long'), {'fs': 100.0, 'gyro': gyro, 'accel': accel}, deg=False)
    alg = allan_analysis.Allan(overlapping=True) if plugin == 'Allan' else allan_analysis.Hadamard()
    had = plugin == 'Hadamard'
    sim = Sim([100.0, 0.0, 0.0], d, ref_frame=0, imu=None, algorithm=alg)
    sim.run(1)
    pre = 'hd_' if had else 'ad_'
    da, dg = (sim.get_data([pre + k])[0]['algo0_0'] for k in ('accel', 'gyro'))
    for dev, x, what in ((da, accel, 'accel'), (dg, gyro, 'gyro')):
        for c in range(3):
            ref = _reference(x[:, c], 100.0, had)
            cls = ref[2]['cls']
            assert np.array_equal(np.isnan(dev[:, c]), cls == 2) and np.all(dev[cls == 1, c] == np.inf), (what, c)
            if (cls == 0).all():
                v, _ = _run(eng, 100.0, x[:, c][None], had)
                assert np.array_equal(dev[:, c], np.sqrt(v[0])), (what, c)
                _check(v[0], x[:, c], ref, 'logged %s %s %d' % (plugin, what, c), (plugin.lower(), 'logged'))
    assert np.isnan(da[:, 2]).all() and np.isinf(dg[:, 1]).all()
