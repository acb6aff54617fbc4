"""The Welch reference (oracle/welch_exact.py) against mpmath at 200 bits, welch_np and scipy; and K11's
algorithm restated in float64 (welch_exact.emulate) within the rigorous bound and the sharp scale U_k over the
grid of tests/test_gpu_welch_edges.py at shorter lengths.  Prints the emulation's worst error/bound and worst
e = max |emulated - exact| / U_k per transform form: 4x the worst e is the threshold the GPU test uses."""
import numpy as np
import pytest

import welch_exact as we
import welch_np as wn

pytestmark = pytest.mark.skipif(not we.have_long_double(),
                                reason='np.longdouble has no 64-bit significand on this platform')

NS = (16, 18, 30, 1002, 1024, 2048, 2050, 4096, 6000, 8190, 8192, 16384)


def _mp_welch(x, fs, N, D, w, mp):
    """welch_np's formula at mp.prec bits: direct DFT of every segment."""
    K, S = wn.segments(len(x), N, D)
    L = N // 2 + 1
    xm = [mp.mpf(float(v)) for v in x]
    wm = [mp.mpf(float(v)) for v in w]
    cs = [[mp.cospi(mp.mpf(2 * k * m) / N) for m in range(N)] for k in range(L)]
    sn = [[mp.sinpi(mp.mpf(2 * k * m) / N) for m in range(N)] for k in range(L)]
    acc = [mp.mpf(0)] * L
    for j in range(K):
        seg = xm[j * S:j * S + N]
        mean = mp.fsum(seg) / N
        y = [(seg[m] - mean) * wm[m] for m in range(N)]
        for k in range(L):
            re = mp.fsum(y[m] * cs[k][m] for m in range(N))
            im = mp.fsum(y[m] * sn[k][m] for m in range(N))
            acc[k] += re * re + im * im
    den = fs * mp.fsum(v * v for v in wm) * K
    return [(1 if k in (0, L - 1) else 2) * acc[k] / den for k in range(L)]


def _series(kind, n, N, rng, scale=1.0):
    t = np.arange(n)
    if kind == 'white':
        return scale * rng.standard_normal(n)
    if kind == 'offset':
        return 1e4 + 1e-9 * rng.standard_normal(n)
    if kind == 'nav':
        return -9.80665 + 1e-5 * rng.standard_normal(n)
    if kind == 'tone_on':
        return np.cos(2 * np.pi * (N // 8) * t / N) + 1e-12 * rng.standard_normal(n)
    if kind == 'tone_off':
        return np.cos(2 * np.pi * (N // 8 + 0.37) * t / N) + 1e-12 * rng.standard_normal(n)
    if kind == 'walk':
        return np.cumsum(rng.standard_normal(n))
    raise ValueError(kind)


@pytest.mark.parametrize('N, D, kind, scale', [
    (16, 8, 'white', 1.0), (18, 9, 'white', 1.0), (20, 5, 'offset', 1.0), (18, 0, 'nav', 1.0),
    (16, 8, 'tone_off', 1.0), (18, 9, 'white', 1e-150), (16, 7, 'white', 1e150), (30, 15, 'tone_on', 1.0)])
def test_reference_against_mpmath(N, D, kind, scale):
    mp = pytest.importorskip('mpmath').mp
    mp.prec = 200
    rng = np.random.default_rng(N * 7 + D)
    n = 3 * N - D + 1
    x = _series(kind, n, N, rng, scale)
    for w in (wn.hann(N), rng.uniform(0.1, 1.0, N)):
        r = we.welch(x, 3.0, N, D, w, need=('psd', 'U'))
        exact = _mp_welch(x, 3.0, N, D, w, mp)
        for k, (got, want) in enumerate(zip(r['psd'], exact)):
            want_f = float(want)
            # the long-double work sits far below U_k (u = 2^-53); the result is rounded once
            tol = 2.0 ** -52 * abs(want_f) + 1e-3 * r['U'][k]
            assert abs(got - want_f) <= tol, (k, got, want_f, tol)


@pytest.mark.parametrize('N, D, n', [(256, 128, 5000), (1000, 300, 7000), (18, 9, 400), (16384, 8192, 70000)])
def test_reference_against_welch_np_and_scipy(N, D, n):
    rng = np.random.default_rng(n)
    x = rng.standard_normal(n) * 0.3 + 2.0
    w = wn.hann(N)
    r = we.welch(x, 50.0, N, D, w, need=('psd', 'U'))
    f, p = wn.welch(x, 50.0, N, D, w)
    # a float64 transform and mean: within a few hundred U_k of the exact PSD
    assert (np.abs(p - r['psd']) <= 300 * r['U']).all(), (np.abs(p - r['psd']) / r['U']).max()
    sig = pytest.importorskip('scipy.signal')
    f2, p2 = sig.welch(x, fs=50.0, window=w, nperseg=N, noverlap=D, detrend='constant')
    assert (np.abs(p2 - r['psd']) <= 300 * r['U']).all(), (np.abs(p2 - r['psd']) / r['U']).max()


def test_non_finite_rule():
    N, D = 64, 32
    x = np.random.default_rng(2).standard_normal(500)
    K, S = wn.segments(500, N, D)
    for bad in (np.nan, np.inf, -np.inf):
        y = x.copy()
        y[S * (K - 1) + N - 1] = bad
        assert np.isnan(we.welch(y, 1.0, N, D, wn.hann(N))['psd']).all()
        y = x.copy()
        y[S * (K - 1) + N:] = bad
        assert np.array_equal(we.welch(y, 1.0, N, D, wn.hann(N))['psd'], we.welch(x, 1.0, N, D, wn.hann(N))['psd'])
    assert (we.welch(np.full(300, 1e305), 1.0, N, D, wn.hann(N))['psd'] == 0.0).all()
    big = we.welch(1e154 * x, 1e-6, N, D, wn.hann(N))['psd']
    assert np.isinf(big).any() and not np.isnan(big).any()


def _grid_cases():
    """(N, D, n, kind, window name) over the GPU grid's forms at CPU-sized lengths."""
    for N in NS:
        for D in sorted({0, N // 2, N - 1, N // 2 - 3 if (N // 2) % 2 == 0 else N // 2}):
            S = N - D
            for n in (N, N + S - 1, N + 5 * S):
                for kind in ('white', 'offset', 'nav', 'tone_on', 'tone_off', 'walk'):
                    if N >= 8190 and (D != N // 2 or kind in ('tone_on', 'walk')):
                        continue
                    yield N, D, n, kind, 'hann'
        D = N // 2
        pl = we.plan(10 ** 9, N, D)
        for K in {pl['Q'] - 1, pl['Q'] + 1, pl['G'] + 1, 2 * pl['G'] - 1} if N <= 1024 else {pl['Q'] + 1}:
            if K >= 1 and K * (N - D) <= 40000:
                yield N, D, D + K * (N - D), 'white', 'rand'


def _window(name, N, rng):
    return wn.hann(N) if name == 'hann' else rng.uniform(0.2, 1.0, N)


def test_emulation_within_the_bound_and_U_on_the_grid():
    worst = {'radix-2': [0.0, 0.0, None], 'bluestein': [0.0, 0.0, None]}
    for N, D, n, kind, wname in _grid_cases():
        rng = np.random.default_rng(N + 7 * D + n)
        x = _series(kind, n, N, rng)
        w = _window(wname, N, rng)
        r = we.welch(x, 2.0, N, D, w, need=('psd', 'U', 'bound'))
        em = we.emulate(x, 2.0, N, D, w)
        err = np.abs(em - r['psd'])
        assert (err <= r['bound']).all(), (N, D, n, kind, (err / r['bound']).max())
        form = 'bluestein' if we.plan(n, N, D)['bluestein'] else 'radix-2'
        b, e = (err / r['bound']).max(), (err / r['U']).max()
        if e > worst[form][1]:
            worst[form][1], worst[form][2] = e, (N, D, n, kind, wname)
        worst[form][0] = max(worst[form][0], b)
    for form, (b, e, case) in worst.items():
        print('emulation %-9s worst error/bound %.3g, worst e %.3g at (N, D, n, data, window) = %s'
              % (form, b, e, case))
    # the GPU thresholds are 4x these; a change of the algorithm that moves them must move the thresholds too
    assert worst['radix-2'][1] <= 42.5 and worst['bluestein'][1] <= 52.0, worst


@pytest.mark.parametrize('mutant', ['mean_ulp', 'half_step_conj', 'chirp_mod_m'])
def test_emulated_mistakes_are_caught(mutant):
    """A mean off by one ulp, the conjugate odd-bin half step and the chirp reduced mod M each exceed 1000 times the
    sharp scale on a case of their form."""
    rng = np.random.default_rng(5)
    N = {'mean_ulp': 256, 'half_step_conj': 256, 'chirp_mod_m': 1002}[mutant]
    x = 1e4 + 1e-9 * rng.standard_normal(4 * N)
    r = we.welch(x, 1.0, N, N // 2, wn.hann(N), need=('psd', 'U'))
    em = we.emulate(x, 1.0, N, N // 2, wn.hann(N), mutant=mutant)
    assert (np.abs(em - r["psd"]) / r["U"]).max() > 1000
