"""The exact overlapping Allan and Hadamard variances (oracle/oallan_exact.py), the reference K4o is held to:
against the definition in Fractions, the fixed-point and long-double oracles, its own two integer paths and the
IEEE class of the definitional sum on a bank of non-finite cases.  Then a NumPy emulation of K4o's arithmetic in
its fixed order, held within the bound of tests/test_gpu_oallan_edges.py before any GPU time is spent.  No GPU."""
from fractions import Fraction

import numpy as np
import pytest

import oallan_exact as ox
import oallan_np as oa
import ohadamard_np as oh

WORST = {}          # form -> worst |emulation - exact| / bound


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nK4o emulation worst |emulated - exact| / bound: ' +
          ', '.join('%s %.3g' % kv for kv in sorted(WORST.items())))


def _float(f):
    try:
        return float(f)
    except OverflowError:
        return np.inf


def _fraction(x, fs, had):
    """The definition in Fractions: every window summed directly, one rounding at the end (finite x)."""
    n = len(x)
    xf = [Fraction(v) for v in x]
    out = []
    for m in oa._grid(n, fs)[0]:
        S = [sum(xf[k:k + m]) for k in range(n - m + 1)]
        if had:
            K = n - 3 * m + 1
            s = sum((S[k + 2 * m] - 2 * S[k + m] + S[k]) ** 2 for k in range(K))
            out.append(_float(s / (6 * m * m * K)))
        else:
            K = n - 2 * m + 1
            s = sum((S[k + m] - S[k]) ** 2 for k in range(K))
            out.append(_float(s / (2 * m * m * K)))
    return np.array(out)


def _series(case, n, rng):
    i = np.arange(n, dtype=np.float64)
    return {'white': rng.standard_normal(n),
            'offset_1e7': 1e7 + rng.standard_normal(n),
            'drift': np.where(i == 0, 0.0, 1e-3 * i + 1e-6 * rng.standard_normal(n)),
            'ramp': 1e4 + 1e-3 * i + 1e-3 * rng.standard_normal(n),
            'quadratic': 2.0 + 1e-3 * i + 1e-5 * i * i + 0.1 * rng.standard_normal(n),
            'walk': np.cumsum(rng.standard_normal(n)),
            'outlier_x0': np.concatenate([[1e6], rng.standard_normal(n - 1)]),
            'step': np.where(i < n // 2, 0.0, 5.0) + rng.standard_normal(n),
            'integer': rng.integers(-2000, 2000, n).astype(np.float64),
            'tiny_1e-150': 1e-150 * rng.standard_normal(n),
            'huge_1e150': 1e150 * rng.standard_normal(n)}[case]


CASES = ['white', 'offset_1e7', 'ramp', 'quadratic', 'walk', 'outlier_x0', 'step', 'integer', 'tiny_1e-150',
         'huge_1e150']


@pytest.mark.parametrize('had', [False, True], ids=['allan', 'hadamard'])
@pytest.mark.parametrize('case', CASES)
def test_exact_against_fractions(case, had):
    n = 100
    x = _series(case, n, np.random.default_rng(len(case)))
    got, tau, info = ox.exact(x, 1.0, had)
    assert len(got) == len(oa._grid(n, 1.0)[0]) > 0 and info['path'] == 'limbs'
    assert np.array_equal(got, _fraction(x, 1.0, had)), (got, _fraction(x, 1.0, had))
    assert np.array_equal(tau, oa._grid(n, 1.0)[1])


def test_exact_across_binades_takes_python_ints():
    """Samples from 1e-140 to 1e140 span ~930 bits: the Python-int path, still equal to the Fractions."""
    rng = np.random.default_rng(3)
    x = rng.standard_normal(60) * 10.0 ** rng.integers(-140, 140, 60)
    for had in (False, True):
        got, _, info = ox.exact(x, 1.0, had)
        assert info['path'] == 'ints'
        assert np.array_equal(got, _fraction(x, 1.0, had))
        with pytest.raises(ValueError):
            ox.exact(x, 1.0, had, path='limbs')


@pytest.mark.parametrize('case', CASES)
def test_limb_and_int_paths_give_the_same_bits(case):
    n = 20011
    x = _series(case, n, np.random.default_rng(7))
    for had in (False, True):
        a, _, ia = ox.exact(x, 1.0, had, path='limbs')
        b, _, ib = ox.exact(x, 1.0, had, path='ints')
        assert np.array_equal(a, b), case
        assert np.array_equal(ia['tmax'], ib['tmax']) or np.allclose(ia['tmax'], ib['tmax'], rtol=1e-15, atol=0)


def test_against_the_fixed_point_hadamard_oracle():
    """ohadamard_var_fixed: exact terms, squares and their sum in long double (64-bit mantissa): within
    ~ (K + 2) 2^-64 of the exact value."""
    rng = np.random.default_rng(5)
    n = 200003
    for x in (1e4 + 1e-3 * np.arange(n) + 1e-3 * rng.standard_normal(n),
              1.5 + 0.25 * rng.random(n),
              1000.0 + rng.integers(-1000, 1000, n) * 2.0 ** -10):
        ex, _ = ox.ohadamard_var(x, 1.0)
        fx, _ = oh.ohadamard_var_fixed(x, 1.0)
        assert np.all(np.abs(fx - ex) <= (n + 2) * 2.0 ** -63 * ex), np.abs(fx / ex - 1).max()


@pytest.mark.parametrize('n', [9000, 5 * 2048 + 1, 7 * 2304 - 1, 90009])
def test_against_the_long_double_oracles(n):
    """Where the long-double prefix holds (white noise on a modest offset), both forms agree to 1e-12."""
    x = np.random.default_rng(n).standard_normal(n) + 0.5
    ex, tau = ox.oallan_var(x, 1.0)
    o, ot = oa.oallan_var(x, 1.0)
    assert np.array_equal(tau, ot) and np.all(np.abs(o / ex - 1.0) <= 1e-12)
    ex, _ = ox.ohadamard_var(x, 1.0)
    o, _ = oh.ohadamard_var(x, 1.0)
    assert np.all(np.abs(o / ex - 1.0) <= 1e-12)


def test_overflowing_prefix_is_inf():
    """x_0 = -1e305 and every other sample +1e305: the shifted prefix passes DBL_MAX, the first term is 2e305 and
    its square over 2 m^2 M is past DBL_MAX at every tau."""
    x = np.full(9 * 2304 + 5, 1e305)
    x[0] = -1e305
    for had in (False, True):
        v, _, info = ox.exact(x, 1.0, had)
        assert np.all(v == np.inf) and np.all(info['cls'] == 0)


def _bank(n):
    rng = np.random.default_rng(n)
    base = rng.standard_normal(n)
    T = 2304
    cases = []
    for spots in ([(0, np.nan)], [(n - 1, np.nan)], [(0, np.inf)], [(0, -np.inf)], [(0, np.inf), (1, -np.inf)],
                  [(n - 1, np.inf)], [(T - 1, np.inf)], [(T, -np.inf)], [(3, np.inf), (4 * T + 7, -np.inf)],
                  [(100, np.inf), (101, np.inf)], [(100, np.inf), (102, np.inf)], [(100, -np.inf), (103, -np.inf)],
                  [(100, np.inf), (107, -np.inf)], [(2 * T + 5, np.inf), (2 * T + 9, np.inf), (2 * T + 30, -np.inf)],
                  [(3, np.nan), (999, np.inf)], [(500, np.inf), (1500, -np.inf), (2500, np.nan)]):
        x = base.copy()
        for i, v in spots:
            if i < n:
                x[i] = v
        cases.append(x)
    return cases


@pytest.mark.parametrize('n', [400, 4 * 2304 + 1001])
def test_non_finite_class_is_the_definitions(n):
    """NaN and +inf exactly where the definition in IEEE arithmetic (oallan_var_brute, ohadamard_var_brute) gives
    them; the finite taus are those of the series with the changed samples left out."""
    for x in _bank(n):
        for had, brute in ((False, oa.oallan_var_brute), (True, oh.ohadamard_var_brute)):
            ex, _, info = ox.exact(x, 1.0, had)
            with np.errstate(invalid='ignore', over='ignore'):
                b, _ = brute(x, 1.0)
            assert np.array_equal(np.isnan(ex), np.isnan(b)), (had, np.nonzero(~np.isfinite(x)), ex, b)
            assert np.array_equal(np.isinf(ex), np.isinf(b)) and not (ex == -np.inf).any()
            assert np.all(np.isfinite(ex) == (info['cls'] == 0))
    for had in (False, True):         # +inf and -inf 7 apart: NaN where a window holds both, +inf below
        both = ox.exact(_bank(n)[12], 1.0, had)[0]
        assert np.isnan(both).any() and np.isinf(both).any()


# ---------------------------------------------------------------------------------------------------------------
# K4o's arithmetic, emulated in NumPy in its fixed order (finite series)
# ---------------------------------------------------------------------------------------------------------------
SCAN_T, SCAN_P, SQ_T, SQ_P = 256, 9, 256, 8


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _quick_two_sum(a, b):
    s = a + b
    return s, b - (s - a)


def _dd_add_d(h, l, b):
    s, e = _two_sum(h, b)
    return _quick_two_sum(s, e + l)


def _dd_add(ah, al, bh, bl):
    s, e = _two_sum(ah, bh)
    return _quick_two_sum(s, e + (al + bl))


def _dd_diff(ah, al, bh, bl):
    s, e = _two_sum(ah, -bh)
    return s, e + (al - bl)


def _fma_sq(t, acc):
    """fma(t, t, acc) rounded once: the exact product (Dekker), then a sum rounded to odd and once to nearest
    (Boldo and Melquiond's emulation of an FMA).  Normal range, no overflow."""
    c = 134217729.0 * t
    th = c - (c - t)
    tl = t - th
    ph = t * t
    pl = ((th * th - ph) + 2.0 * th * tl) + tl * tl
    sh, sl = _two_sum(acc, ph)
    v, ve = _two_sum(sl, pl)                     # v rounded to odd: step off an even last bit toward the error
    bits = v.view(np.int64)
    even = (bits & 1) == 0
    v = np.where((ve != 0.0) & even, np.nextafter(v, np.where(ve > 0.0, np.inf, -np.inf)), v)
    return sh + v


def _butterfly(v):
    """The 5-step xor butterfly over the last axis (32 lanes); every lane ends with lane 0's value."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., lanes ^ o]
    return v[..., 0]


def k4o_emulate(x, fs, had):
    """K4o's five passes on one finite series, operation for operation (tiles, threads, lanes in its order)."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    mult, tau = oa._grid(n, fs)
    tiles = -(-n // (SCAN_T * SCAN_P))
    y = np.zeros(tiles * SCAN_T * SCAN_P)
    y[:n] = x - x[0]
    valid = (np.arange(len(y)) < n).reshape(tiles, SCAN_T, SCAN_P)
    y = y.reshape(tiles, SCAN_T, SCAN_P)
    # the thread-serial runs (pass 1 and pass 3 compute the same ones)
    loc = np.zeros((2,) + y.shape)
    h = np.zeros((tiles, SCAN_T))
    lo = np.zeros((tiles, SCAN_T))
    for q in range(SCAN_P):
        nh, nl = _dd_add_d(h, lo, y[:, :, q])
        h, lo = np.where(valid[:, :, q], nh, h), np.where(valid[:, :, q], nl, lo)
        loc[0, :, :, q], loc[1, :, :, q] = h, lo
    # Hillis-Steele over the 256 thread totals
    sh, sl = h.copy(), lo.copy()
    o = 1
    while o < SCAN_T:
        nh, nl = _dd_add(sh[:, :-o], sl[:, :-o], sh[:, o:], sl[:, o:])
        sh, sl = sh.copy(), sl.copy()
        sh[:, o:], sl[:, o:] = nh, nl
        o <<= 1
    # pass 2: the exclusive carry of every tile, one tile after the other
    ch, cl = np.zeros(tiles), np.zeros(tiles)
    rh = rl = 0.0
    for t in range(tiles):
        ch[t], cl[t] = rh, rl
        rh, rl = _dd_add(np.float64(rh), np.float64(rl), sh[t, -1], sl[t, -1])
    # pass 3
    eh = np.repeat(ch[:, None], SCAN_T, 1)
    el = np.repeat(cl[:, None], SCAN_T, 1)
    a, b = _dd_add(eh[:, 1:], el[:, 1:], sh[:, :-1], sl[:, :-1])
    eh[:, 1:], el[:, 1:] = a, b
    Ch, Cl = _dd_add(eh[:, :, None], el[:, :, None], loc[0], loc[1])
    C = np.zeros((2, n + 1))
    C[0, 1:], C[1, 1:] = Ch.reshape(-1)[:n], Cl.reshape(-1)[:n]
    # pass 4: the terms; offsets k = tile 2048 + q 256 + tid, FMA chains over q; lanes, warps; pass 5
    sq_tiles = -(-n // (SQ_T * SQ_P))
    w = 3 if had else 2
    out = np.zeros(len(mult))
    for i, m in enumerate(mult):
        K = n - w * m + 1
        c = [C[:, j * m:j * m + K] for j in range(w + 1)]
        if had:
            s0 = _dd_diff(c[1][0], c[1][1], c[0][0], c[0][1])
            s1 = _dd_diff(c[2][0], c[2][1], c[1][0], c[1][1])
            s2 = _dd_diff(c[3][0], c[3][1], c[2][0], c[2][1])
            t = ((s2[0] - s1[0]) - (s1[0] - s0[0])) + ((s2[1] - s1[1]) - (s1[1] - s0[1]))
        else:
            da = _dd_diff(c[1][0], c[1][1], c[0][0], c[0][1])
            db = _dd_diff(c[2][0], c[2][1], c[0][0], c[0][1])
            t = (db[0] - 2.0 * da[0]) + (db[1] - 2.0 * da[1])
        tt = np.zeros(sq_tiles * SQ_T * SQ_P)
        tt[:K] = t
        tt = tt.reshape(sq_tiles, SQ_P, SQ_T)
        acc = np.zeros((sq_tiles, SQ_T))
        for q in range(SQ_P):
            acc = _fma_sq(tt[:, q], acc)
        warp = _butterfly(acc.reshape(sq_tiles, SQ_T // 32, 32))
        part = np.zeros(sq_tiles)
        for wi in range(SQ_T // 32):
            part = part + warp[:, wi]
        lanes = np.zeros(32)
        for t0 in range(0, sq_tiles, 32):
            seg = part[t0:t0 + 32]
            lanes[:len(seg)] = lanes[:len(seg)] + seg
        v = _butterfly(lanes)
        mf = np.float64(m)
        out[i] = v / ((6.0 if had else 2.0) * mf * mf * np.float64(K))
    return out, tau


def test_fma_emulation_rounds_once():
    rng = np.random.default_rng(1)
    t = rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 30, 4000)
    acc = np.abs(rng.standard_normal(4000)) * 2.0 ** rng.integers(-60, 60, 4000)
    got = _fma_sq(t, acc)
    want = np.array([float(Fraction(a) * Fraction(a) + Fraction(c)) for a, c in zip(t, acc)])
    assert np.array_equal(got, want)
    assert not np.array_equal(got, t * t + acc)


EMU_CASES = [('white', 9000), ('drift', 11519), ('offset_1e4', 5 * 2048 + 1), ('offset_1e7', 7 * 2304 - 1), ('ramp', 100000),
             ('quadratic', 50004), ('walk', 30000), ('outlier_x0', 2304 * 4), ('integer', 2048 * 3 + 2),
             ('huge_1e150', 4608)]


@pytest.mark.parametrize('had', [False, True], ids=['allan', 'hadamard'])
@pytest.mark.parametrize('case,n', EMU_CASES)
def test_emulation_within_the_bound(case, n, had):
    rng = np.random.default_rng(n)
    x = (1e4 + rng.standard_normal(n)) if case == 'offset_1e4' else _series(case, n, rng)
    ex, tau, info, bound = ox.k4o_bound(x, 1.0, had)
    got, gt = k4o_emulate(x, 1.0, had)
    assert np.array_equal(gt, tau)
    err = np.abs(got - ex)
    assert np.all(err <= bound), (case, np.nonzero(err > bound), (err / bound).max())
    if case == 'integer':
        assert np.array_equal(got, ex)
    key = 'hadamard' if had else 'allan'
    WORST[key] = max(WORST.get(key, 0.0), float((err / bound).max()))


def test_emulation_of_an_overflowing_prefix_gives_nan():
    """What K4o's finite form computes when the shifted prefix overflows: two_sum of an infinite sum is NaN, and
    NaN reaches every tau.  oallan_final_kernel reports such a finite-sample series as +inf, the exact value."""
    x = np.full(3 * 2304, 1e305)
    x[0] = -1e305
    with np.errstate(invalid='ignore', over='ignore'):
        got, _ = k4o_emulate(x, 1.0, False)
    assert np.all(np.isnan(got))
    assert np.all(ox.oallan_var(x, 1.0)[0] == np.inf)
