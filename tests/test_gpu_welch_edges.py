"""Welch PSD (K11) on the GPU against the exact reference (oracle/welch_exact.py) on every transform form, at its
shape, chunk, magnitude and non-finite edges, and through every front end.

Every finite bin is held to two criteria (welch_exact's docstring defines both):
  * |K11_k - P_k| <= bound_k, the rigorous bound on K11's rounding in its own operation order: the compensated
    mean's summation depth, the subtraction and window product, the radix-2 transform (Higham Thm 24.2) or the
    Bluestein pipeline (chirp products, bhat's own transform error, the pointwise product, the second
    transform), the split step, |.|^2, the in-chunk, slot-tree and chunk-order sums, c_k and the scale;
  * e = max_k |K11_k - P_k| / U_k <= TAU[form], U_k the first-order size of a u-relative rounding spread over
    each segment plus one rounding of the result.  A worst-case FFT bound is ~sqrt(N) looser than what random
    data shows, so the bound alone would miss a subtle mistake at N = 16384; U_k does not.
TAU is 4x the worst e of K11's algorithm emulated in float64 over the CPU grid (tests/test_cpu_welch_exact.py:
radix-2 42.2 on an off-bin tone at N = 16384, Bluestein 51.9 on a random walk at N = 6000, times 4 rounded up).
The worst e sits in bins far below u ||y||: there the error is |dX|^2 against U's second-order d^2.  K11's bits
are deterministic for fixed inputs, so the check cannot be flaky; a device e above TAU is a finding to explain,
not a reason to raise TAU.  U_k and the bound are long double, so neither overflows at the top of the range.

A result is +inf only where the exact PSD, or it plus the bound, reaches DBL_MAX, or where one segment's own PSD
exceeds 16 DBL_MAX (welch_kernel.cuh, Range); a finite result must be within the bound, so a PSD above DBL_MAX
by more than the bound must come back +inf; NaN only from a non-finite sample in a used segment.
The worst error/bound and e per form are printed at the end of the module (pytest -s)."""
import numpy as np
import pytest

import welch_exact as we
import welch_np as wn
from conftest import write_logged_dir

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not we.have_long_double(), reason='np.longdouble has no 64-bit significand')]
torch = pytest.importorskip('torch')

TAU = {'radix-2': 170.0, 'bluestein': 208.0}
NS = (16, 18, 30, 1002, 1024, 2048, 2050, 4096, 6000, 8190, 8192, 16384)
_WORST = {'radix-2': [0.0, None, 0.0, None], 'bluestein': [0.0, None, 0.0, None]}


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _welch(eng, fs, x, N, D, window):
    x = np.ascontiguousarray(x, dtype=np.float64)
    psd, freq = eng.welch(fs, eng.to_device(x), x.shape[1], x.shape[0], N, D, np.asarray(window, dtype=np.float64))
    torch.cuda.synchronize()
    return psd.cpu().numpy(), freq.cpu().numpy()


def _check(got, x, fs, N, D, w, what):
    """got against the exact PSD of x: the bound, U_k, and the overflow and NaN rules."""
    r = we.welch(x, fs, N, D, w, need=('psd', 'U', 'bound'))
    ref = r['psd']
    if np.isnan(ref).any():
        assert np.isnan(got).all(), what
        return
    assert not np.isnan(got).any(), '%s: NaN from finite samples' % what
    big = np.longdouble(np.finfo(np.float64).max)
    exact, bnd, U = r['psd_ld'], r['bound'], r['U']
    # +inf only where the exact PSD, or its rounding bound, reaches DBL_MAX, or where one segment's own PSD is
    # above 16 DBL_MAX (welch_kernel.cuh, Range); a finite result within the bound everywhere, so a finite
    # result where the PSD exceeds DBL_MAX by more than the bound fails too
    ginf = np.isinf(got)
    ok_inf = (exact + bnd >= big) | (r['segmax'] > 16 * big)
    assert not (ginf & ~ok_inf).any(), '%s: +inf where the PSD is finite (%d bins)' % (what, (ginf & ~ok_inf).sum())
    fin = ~ginf
    err = np.abs(got[fin].astype(np.longdouble) - exact[fin])
    assert (err <= bnd[fin]).all(), '%s: worst error/bound %.3g' % (what, float((err / bnd[fin]).max()))
    # the sharp scale where the exact PSD is a float64
    sharp = exact[fin] <= big
    err, bnd, U = err[sharp], bnd[fin][sharp], U[fin][sharp]
    assert (err[U == 0] == 0).all(), what
    e = float((err[U > 0] / U[U > 0]).max()) if (U > 0).any() else 0.0
    form = 'bluestein' if we.plan(x.size, N, D)['bluestein'] else 'radix-2'
    b = float((err[bnd > 0] / bnd[bnd > 0]).max()) if (bnd > 0).any() else 0.0
    wst = _WORST[form]
    if b > wst[0]:
        wst[0], wst[1] = b, what
    if e > wst[2]:
        wst[2], wst[3] = e, what
    assert e <= TAU[form], '%s: e = %.3g > TAU = %g' % (what, e, TAU[form])


def _series(kind, n, N, rng):
    t = np.arange(n)
    return {'white': lambda: rng.standard_normal(n),
            'offset': lambda: 1e4 + 1e-9 * rng.standard_normal(n),
            'nav': lambda: -9.80665 + 1e-5 * rng.standard_normal(n),
            'tone_on': lambda: np.cos(2 * np.pi * (N // 8) * t / N) + 1e-12 * rng.standard_normal(n),
            'tone_off': lambda: np.cos(2 * np.pi * (N // 8 + 0.37) * t / N) + 1e-12 * rng.standard_normal(n),
            'walk': lambda: np.cumsum(rng.standard_normal(n)),
            'const': lambda: np.full(n, 1.0 / 3.0)}[kind]()


KINDS = ('white', 'offset', 'nav', 'tone_on', 'tone_off', 'walk', 'const')


def _windows(N, rng):
    wz = rng.uniform(0.2, 1.0, N)
    wz[::7] = 0.0
    return {'hann': wn.hann(N), 'boxcar': np.ones(N), 'rand': rng.uniform(0.2, 1.0, N), 'zeros': wz}


@pytest.mark.parametrize('N', NS)
def test_forms_overlaps_and_data(eng, N):
    """Every data kind under Hann at D in {0, N/2, N-1, odd}, n in {N, N + S - 1}; every window on white noise."""
    rng = np.random.default_rng(N)
    fs = 200.0
    odd = N // 2 - 3 if (N // 2) % 2 == 0 else N // 2
    for D in sorted({0, N // 2, N - 1, odd}):
        S = N - D
        for n in (N, N + S - 1):
            xs = np.stack([_series(k, n, N, rng) for k in KINDS])
            psd, freq = _welch(eng, fs, xs, N, D, wn.hann(N))
            assert np.array_equal(freq, np.fft.rfftfreq(N, 1.0 / fs))
            for s, kind in enumerate(KINDS):
                _check(psd[s], xs[s], fs, N, D, wn.hann(N), 'N=%d D=%d n=%d %s hann' % (N, D, n, kind))
            if D == N // 2:
                for name, w in _windows(N, rng).items():
                    p, _ = _welch(eng, fs, xs[:1], N, D, w)
                    _check(p[0], xs[0], fs, N, D, w, 'N=%d D=%d n=%d white %s' % (N, D, n, name))


@pytest.mark.parametrize('N', NS)
def test_chunk_and_round_edges(eng, N):
    """K = Q - 1, Q, Q + 1 segments per chunk, K mod G in {0, 1, G - 1}, and K >= 3Q (several chunks)."""
    D = N // 2
    pl = we.plan(10 ** 12, N, D)
    Q, G = pl['Q'], pl['G']
    Ks = sorted({Q - 1, Q, Q + 1, 3 * Q + 1, 2 * G, 2 * G + 1, 3 * G - 1} - {0})
    rng = np.random.default_rng(N + 1)
    for K in Ks:
        n = D + K * (N - D)
        xs = np.stack([rng.standard_normal(n), -9.80665 + 1e-5 * rng.standard_normal(n)])
        psd, _ = _welch(eng, 10.0, xs, N, D, wn.hann(N))
        for s in range(2):
            _check(psd[s], xs[s], 10.0, N, D, wn.hann(N), 'N=%d K=%d (Q=%d G=%d) series %d' % (N, K, Q, G, s))


@pytest.mark.parametrize('N', (1024, 1002, 16384, 8190))
def test_exact_invariants(eng, N):
    """psd(-x) = psd(x); psd(2^e x) = 2^(2e) psd(x); psd at fs 2^e = 2^-e psd; psd with 2^e w = psd, bit for
    bit for e across +-450, where nothing over- or underflows."""
    rng = np.random.default_rng(N + 2)
    n = 3 * N
    x = rng.standard_normal(n) + 0.5
    w = wn.hann(N)
    base, _ = _welch(eng, 1.0, x[None], N, N // 2, w)
    neg, _ = _welch(eng, 1.0, -x[None], N, N // 2, w)
    assert np.array_equal(neg, base)
    for e in (-450, -200, -17, 3, 200, 450):
        p, _ = _welch(eng, 1.0, np.ldexp(x, e)[None], N, N // 2, w)
        assert np.array_equal(p, np.ldexp(base, 2 * e)), ('x', e)
        p, _ = _welch(eng, np.ldexp(1.0, e), x[None], N, N // 2, w)
        assert np.array_equal(p, np.ldexp(base, -e)), ('fs', e)
        p, _ = _welch(eng, 1.0, x[None], N, N // 2, np.ldexp(w, e))
        assert np.array_equal(p, base), ('w', e)
    if N & (N - 1) == 0:
        for c in (0.75, -3.0, 1e305, -1e-300):
            p, _ = _welch(eng, 1.0, np.full((1, n), c), N, N // 2, w)
            assert (p == 0.0).all(), c


@pytest.mark.parametrize('N', (16384, 8190, 1024, 18))
def test_magnitudes_and_rates(eng, N):
    """sigma from 1e-150 to 1e152 on both forms, an offset of 1e305 with noise, fs in {1e-6, 1, 1e6}: within the
    bound where the exact PSD is finite, +inf only where it exceeds DBL_MAX, never NaN.  At fs = 1e-6 sigma =
    1e151 puts the PSD astride DBL_MAX, with segments whose own share is above it; constants of 1e305 and
    1e305/3 give exactly 0; tones up to 1.5e307 and a series alternating +-1.5e308, whose transforms would
    overflow unscaled, give +inf, not NaN."""
    rng = np.random.default_rng(N + 3)
    D = N // 2
    n = D + 101 * (N - D) if N >= 8190 else D + 1000 * (N - D)
    z = rng.standard_normal(n)
    rows, names = [], []
    for sig in (1e-150, 1e-50, 1.0, 1e50, 1e149, 1e150, 1e151, 1e152, 1e154):
        rows.append(sig * z)
        names.append('sigma=%g' % sig)
    rows.append(1e305 + 1e291 * z)
    names.append('1e305 + 1e291 z')
    rows.append(np.full(n, 1e305))
    names.append('1e305 constant')
    rows.append(np.full(n, 1e305 / 3))
    names.append('1e305/3 constant')
    t = np.arange(n)
    for amp in (1e150, 1e305, 1.5e307):
        rows.append(amp * np.cos(2 * np.pi * (N // 8) * t / N))
        names.append('tone %g' % amp)
    rows.append(np.where(t % 2 == 0, 1.5e308, -1.5e308))
    names.append('+-1.5e308 alternating')
    xs = np.stack(rows)
    for fs in (1e-6, 1.0, 1e6):
        psd, _ = _welch(eng, fs, xs, N, D, wn.hann(N))
        for s, name in enumerate(names):
            if s == 0 and fs > 1.0:
                # a PSD of 2e-306, with fs sum w^2 up to 6e9: K11's scaled terms are subnormal there, the range
                # it gives up for headroom at the top (welch_kernel.cuh, Range)
                continue
            _check(psd[s], xs[s], fs, N, D, wn.hann(N), 'N=%d fs=%g %s' % (N, fs, name))


def test_non_finite_samples(eng):
    """NaN and +-inf at the first and last used sample of a segment, in a chunk other than the first, and past
    the last segment."""
    N, D = 256, 128
    pl = we.plan(10 ** 9, N, D)
    K = pl['Q'] + 500
    n = D + K * (N - D) + 77
    S = N - D
    base = np.random.default_rng(4).standard_normal(n)
    last = S * (K - 1) + N
    rows = [base]
    for bad in (np.nan, np.inf, -np.inf):
        for i in (0, S * 3, S * 3 + N - 1, S * (pl['Q'] + 10) + 5, last - 1, last, n - 1):
            y = base.copy()
            y[i] = bad
            rows.append(y)
    xs = np.stack(rows)
    psd, _ = _welch(eng, 5.0, xs, N, D, wn.hann(N))
    for s in range(xs.shape[0]):
        _check(psd[s], xs[s], 5.0, N, D, wn.hann(N), 'non-finite row %d' % s)


def test_front_ends(eng, tmp_path):
    """The interleaved (n, 3) layout, a 1000-series batch, Psd().run_batch and a logged directory, each against
    the exact reference."""
    from gnss_ins_sim_b200.psd_analysis import Psd
    from gnss_ins_sim_b200.sim import Sim
    rng = np.random.default_rng(6)
    n, fs, N = 20000, 100.0, 1002
    tri = rng.standard_normal((n, 3)) * np.array([1e-3, 0.3, 1e-5]) + np.array([0.0, 5.0, -9.80665])
    p, _ = eng.welch(fs, eng.to_device(tri[None]), n, 3, N, N // 2, wn.hann(N), inner=3, outer_stride=3 * n,
                     sample_stride=3)
    p = p.cpu().numpy()
    for c in range(3):
        _check(p[c], tri[:, c], fs, N, N // 2, wn.hann(N), 'interleaved axis %d' % c)
    big = rng.standard_normal((1000, 2048)) * 1e-3 + 9.8
    pb, _ = _welch(eng, fs, big, 256, 128, wn.hann(256))
    for s in (0, 1, 517, 999):
        _check(pb[s], big[s], fs, 256, 128, wn.hann(256), 'batch series %d' % s)
    gyro = 1e-4 * rng.standard_normal((2, n, 3))
    accel = 1e-5 * rng.standard_normal((2, n, 3)) + np.array([0.0, 0.0, -9.80665])
    f, pa, pg = Psd(nperseg=2048).run_batch(fs, accel, gyro)
    for r in range(2):
        for c in range(3):
            _check(pa[r][:, c], accel[r, :, c], fs, 2048, 1024, wn.hann(2048), 'run_batch accel %d %d' % (r, c))
            _check(pg[r][:, c], gyro[r, :, c], fs, 2048, 1024, wn.hann(2048), 'run_batch gyro %d %d' % (r, c))
    d = write_logged_dir(str(tmp_path / 'logged'), {'fs': fs, 'gyro': gyro[0], 'accel': accel[0]}, deg=False)
    sim = Sim([fs, 0.0, 0.0], d, ref_frame=0, imu=None, algorithm=Psd(nperseg=2048))
    sim.run(1)
    a = sim.get_data(['psd_accel'])[0]['algo0_0']
    for c in range(3):
        _check(a[:, c], accel[0, :, c], fs, 2048, 1024, wn.hann(2048), 'logged accel %d' % c)


def test_config4_length_channel(eng):
    """One accelerometer z channel at config-4 length (14.4 M samples @400 Hz), K1's own draw, N = 16384."""
    from gnss_ins_sim_b200 import imu_model
    n, fs, N = 14400000, 400.0, 16384
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    ref_gyro = eng.to_device(np.zeros((n, 3)))
    ref_accel = eng.to_device(np.tile([0.0, 0.0, -9.8], (n, 1)))
    gyro, accel = eng.imu_noise(fs, 1, ref_gyro, ref_accel, imu.gyro_err, imu.accel_err, 5,
                                layout=eng.LAYOUT_CHANNEL_MAJOR)
    z = accel[0, 2:3].contiguous()
    psd, _ = eng.welch(fs, z, n, 1, N, N // 2, wn.hann(N))
    psd, z = psd.cpu().numpy()[0], z.cpu().numpy()[0]
    del gyro, accel, ref_gyro, ref_accel
    _check(psd, z, fs, N, N // 2, wn.hann(N), 'config-4 accel z')


def test_zz_report():
    """The worst error/bound and e per form over this module (run with -s to see them)."""
    for form, (b, bc, e, ec) in _WORST.items():
        print('K11 %-9s worst error/bound %.3g (%s); worst e %.3g (%s), TAU %g' % (form, b, bc, e, ec, TAU[form]))
