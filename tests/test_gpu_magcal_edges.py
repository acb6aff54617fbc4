"""K10, the magnetometer calibration, on the GPU against the exact reference (oracle/magcal_exact.py) at its segment,
addressing, conditioning, near-degenerate, magnitude and non-finite edges.

The bound.  magcal_exact.calibrate gives, per output, a first-order bound on K10's rounding in K10's own order:
each moment's sum carries gamma(depth) sum |terms| with depth = ceil(L / 256) per thread + 5 butterfly steps + 7
warp additions + 2 segment additions (plus 1, 3 or 5 roundings of a term); each Gaussian elimination carries
its formation error and the componentwise backward error gamma(3n) |L||U| through |A^-1| (the 4x4 system at
K10's equilibration); the extremes gamma(3) max_k sum |O_i||m_k| (a max is 1-Lipschitz in O); the range ratios,
S = diag(s) O and the final sums and square root their own roundings.  Every perturbation is carried to the
outputs by the exact Jacobian of the pipeline (mpmath), and 1.25 x the sum covers the second-order terms while the
first-order bound is below 1e-3 relative.  mag_cal and the generated form's err get bounds from those of O, s,
S and hard iron plus their own roundings.  The bound grows like cond(M^T M) u, as K10's error does.

Classes: 'singular' (a non-finite sample, an exactly singular plane or sphere system, a zero range) must give NaN
in all 13 outputs; 'regular' (every exact relative pivot above 1e-11) must give a finite result within the bound;
'band' may give either.  K10 is deterministic, so none of this can be flaky.

Magnitudes: the sphere fit is equilibrated by a power of two, so wherever the moments stay in range the result
scales with the samples bit for bit; outside, all 13 outputs are NaN.  Non-finite samples: all 13 outputs and
the run's mag_cal rows are NaN, and the other runs of the batch are unchanged bit for bit.
The worst error / bound per group is printed at the end of the module (pytest -s)."""
import ctypes

import numpy as np
import pytest

import magcal_exact as me
import magcal_np as mc
from test_cpu_magcal_exact import rotations, conditioning_cases, within, check_against_exact

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')
_WORST = {}
SIGMAS = tuple(10.0 ** (-k / 2) for k in range(4, 27)) + (0.0,)     # off-plane noise, uT


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


@pytest.fixture(scope='module', autouse=True)
def report():
    yield
    print('\nK10 worst error / bound per group:')
    for g, (w, what) in sorted(_WORST.items()):
        print('  %-14s %.3g  (%s)' % (g, w, what))


def _note(group, w, what):
    if w >= _WORST.get(group, (-1.0, None))[0]:
        _WORST[group] = (w, what)


def _fed(eng, mag, seg, want_cal=True):
    """K10's fed form on mag [R, n, 3] or [n, 3]: (S [R, 3, 3], hard [R, 4], mag_cal [R, L, 3])."""
    mag = np.asarray(mag, dtype=np.float64)
    if mag.ndim == 2:
        mag = mag[None]
    res = eng.mag_calibrate(np.asarray(seg), eng.to_device(np.ascontiguousarray(mag)), want_cal=want_cal)
    torch.cuda.synchronize()
    cal = res.mag_cal.cpu().numpy() if want_cal else None
    return res.soft_iron.cpu().numpy().reshape(-1, 3, 3), res.hard_iron.cpu().numpy(), cal


def _fed_raw(mag_dev, R, n, seg, run_stride, sample_stride):
    """The C ABI's fed form on a device tensor with explicit strides."""
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    s = np.ascontiguousarray(np.asarray(seg).reshape(-1), dtype=np.int64)
    L = sum(b - a for a, b in np.asarray(seg))
    si = torch.empty((R, 9), dtype=torch.float64, device='cuda')
    hi = torch.empty((R, 4), dtype=torch.float64, device='cuda')
    cal = torch.empty((R, L, 3), dtype=torch.float64, device='cuda')
    D = lambda t: ctypes.c_void_p(t.data_ptr())        # noqa: E731
    assert lib.b2ins_magcal_fed_f64(R, n, s.ctypes.data_as(_lib.c_int64_p), D(mag_dev), run_stride, sample_stride,
                                    D(si), D(hi), D(cal), None) == _lib.OK
    torch.cuda.synchronize()
    return si.cpu().numpy().reshape(R, 3, 3), hi.cpu().numpy(), cal.cpu().numpy()


def _hold(group, what, S, h, cal, mag, seg, model=None, err=None, r=None):
    """One run against the exact reference on its class; cal and err within their bounds."""
    if r is None:
        r = me.calibrate(mag, seg, want_cal=cal is not None, model=model)
    w = check_against_exact(S, h, r, what)
    if np.isfinite(S).all():
        if cal is not None:
            w = max(w, within(cal, r['mag_cal'].astype(np.float64), r['b_cal']))
        if err is not None:
            w = max(w, within(err, r['err'], r['b_err']))
        assert w <= 1.0, '%s: error / bound %.3g' % (what, w)
    elif cal is not None:
        assert np.isnan(cal).all(), '%s: mag_cal of a NaN run' % what
    _note(group, w, what)
    return r


@pytest.mark.parametrize('L', [3, 31, 32, 33, 255, 256, 257, 511, 8193, 100007])
def test_segment_lengths(eng, L):
    sweep = 0.5 if L == 3 else 2.2
    mag, seg = rotations(L=(L, L, L), seed=L % 1000, sweep=sweep)[:2]
    S, h, cal = _fed(eng, mag, seg, want_cal=L <= 8193)
    _hold('segments', 'L = %d' % L, S[0], h[0], None if cal is None else cal[0], mag, seg)


def test_segment_placement(eng):
    mag, _ = rotations(L=(300, 300, 300), seed=31)[:2]
    pad = np.concatenate([np.full((17, 3), 7.0), mag, np.full((40, 3), -3.0)])
    n = pad.shape[0]
    cases = {
        'z y x': (mag[::-1].copy(), ((600, 900), (300, 600), (0, 300))),
        'overlapping': (mag, ((0, 400), (250, 650), (550, 900))),
        'adjacent in the middle': (pad, ((17, 317), (317, 617), (617, 917))),
        'x ends at the last row': (np.concatenate([mag[300:], mag[:300]]), ((600, 900), (0, 300), (300, 600))),
    }
    assert cases['adjacent in the middle'][1][2][1] < n
    for what, (m, seg) in cases.items():
        S, h, cal = _fed(eng, m, seg)
        _hold('segments', what, S[0], h[0], cal[0], m, seg)


def test_strides_and_batches(eng):
    """sample_stride 9 (a view of a nine-axis log), run_stride != 3 n, run_stride 0 (every run the same bits),
    and batches of 1, 7, 1000 and 65 537 runs: each run as it is alone, and a sample held to the exact result."""
    L = 64
    n = 3 * L
    runs = [rotations(L=(L, L, L), seed=100 + r)[0] for r in range(1000)]
    seg = ((0, L), (L, 2 * L), (2 * L, 3 * L))
    nine = np.zeros((7, n, 9))
    nine[:, :, 3:6] = np.stack(runs[:7])
    nine[:, :, 0:3] = 1e300
    nine[:, :, 6:9] = np.nan
    dev = torch.from_numpy(nine).cuda()
    S9, h9, c9 = _fed_raw(dev[:, :, 3:], 7, n, seg, 9 * n, 9)
    # run_stride 3 n + 5 (padding between runs)
    padded = np.full((7, 3 * n + 5), np.nan)
    padded[:, :3 * n] = np.stack(runs[:7]).reshape(7, -1)
    Sp, hp, cp = _fed_raw(torch.from_numpy(padded).cuda(), 7, n, seg, 3 * n + 5, 3)
    for R in (1, 7, 1000):
        S, h, cal = _fed(eng, np.stack(runs[:R]), seg)
        for r in sorted({0, R // 2, R - 1}):
            _hold('addressing', 'R = %d run %d' % (R, r), S[r], h[r], cal[r], runs[r], seg)
        for r in range(0, R, max(1, R // 16)):
            S1, h1, c1 = _fed(eng, runs[r], seg)
            assert np.array_equal(S1[0], S[r]) and np.array_equal(h1[0], h[r]) and np.array_equal(c1[0], cal[r])
        if R == 7:
            for a, b in ((S9, S), (h9, h), (c9, cal), (Sp, S), (hp, h), (cp, cal)):
                assert np.array_equal(a, b)
    # run_stride 0: 65 537 runs of the same samples give the same bits
    one = torch.from_numpy(np.ascontiguousarray(runs[0])).cuda()
    S0, h0, c0 = _fed_raw(one, 65537, n, seg, 0, 3)
    S1, h1, c1 = _fed(eng, runs[0], seg)
    assert (S0 == S1[0]).all() and (h0 == h1[0]).all() and (c0 == c1[0]).all()


def test_generated_form_across_the_run_id_high_word(eng):
    """The generated form with run_offset across 2^32 (the high word of the Philox run id): K8's samples at the
    same offsets, calibrated exactly, with err within its bound; and the runs differ from those 2^32 below."""
    L = 500
    ref, seg = rotations(L=(L, L, L), hard=0.0, noise=0.0, seed=41)[:2]
    si = np.eye(3) + 0.03 * np.random.default_rng(42).standard_normal((3, 3))
    err = {'si': si, 'hi': np.array([8.0, -3.0, 5.0]), 'std': np.full(3, 0.2)}
    off = 2 ** 32 - 2
    refd = eng.to_device(ref)
    gen = eng.mag_calibrate_mc(4, seg, refd, err, 77, run_offset=off)
    low = eng.mag_calibrate_mc(4, seg, refd, err, 77, run_offset=off - 2 ** 32)
    mag = eng.mag_noise(4, refd, err, 77, run_offset=off).cpu().numpy()
    S, h, e = (t.cpu().numpy() for t in (gen.soft_iron, gen.hard_iron, gen.err))
    b = np.linalg.norm(ref[0])
    for r in range(4):
        _hold('generated', 'run %d + %d' % (off, r), S[r].reshape(3, 3), h[r], None, mag[r], seg,
              model=(si, err['hi'], b), err=e[r])
    assert not np.array_equal(low.soft_iron.cpu().numpy()[2:], S[2:])


def test_conditioning(eng):
    cases = list(conditioning_cases())
    batch = np.stack([m for _, m, _, _ in cases])
    seg = cases[0][2]
    assert all(c[2] == seg for c in cases)
    S, h, cal = _fed(eng, batch, seg)
    for i, (what, mag, _, model) in enumerate(cases):
        _hold('conditioning', what, S[i], h[i], cal[i], mag, seg)


def test_near_degenerate(eng):
    """A segment in the plane x = 0 with off-plane noise swept through the pivot band, a constant segment, a
    plane through the origin, collinear samples, and a zero range (the x and y segments in one plane)."""
    L = 300
    base, seg = rotations(L=(L, L, L), hard=0.0, noise=0.0, seed=51)[:2]
    ang = np.linspace(0.0, 2.2 * np.pi, L)
    circle = np.stack([np.zeros(L), 40 * np.cos(ang), 40 * np.sin(ang)], 1)
    rng = np.random.default_rng(52)
    cases = []
    for sig in SIGMAS:
        m = base.copy()
        m[0:L] = circle + np.stack([sig * rng.standard_normal(L), np.zeros(L), np.zeros(L)], 1)
        cases.append(('plane through 0, noise %g' % sig, m))
    m = base.copy()
    m[L:2 * L] = m[L]
    cases.append(('constant segment', m))
    m = base.copy()
    m[2 * L:3 * L] = np.outer(np.arange(L) - L // 2, [3.0, 4.0, 5.0]) / 64.0 + [1.0, 2.0, -7.0]
    cases.append(('collinear', m))
    m = base.copy()
    m[0:L] = circle + [5.0, 0.0, 0.0]
    m[L:2 * L] = circle[::-1] + [5.0, 0.0, 0.0]
    cases.append(('zero range', m))
    S, h, cal = _fed(eng, np.stack([c[1] for c in cases]), seg)
    classes = []
    for i, (what, mag) in enumerate(cases):
        r = _hold('degenerate', what, S[i], h[i], cal[i], mag, seg)
        classes.append(r['cls'])
    assert classes[-3:] == ['singular'] * 3 and classes[0] == 'regular' and classes[len(SIGMAS) - 1] == 'singular', classes
    assert 'band' in classes, classes


def test_magnitudes(eng):
    """The case scaled by 2^k, k = -360 ... 350: bit for bit 2^k times k = 0 wherever the moments stay in range
    (K10's formulation emulated in float64 decides where), all 13 outputs NaN outside."""
    mag, seg = rotations(seed=61)[:2]
    ks = list(range(-360, 351, 10))
    S, h, cal = _fed(eng, np.stack([mag * 2.0 ** k for k in ks]), seg)
    i0 = ks.index(0)
    held = 0
    for i, k in enumerate(ks):
        eS, eh = mc.calibrate_moments(mag * 2.0 ** k, seg, order='kernel')
        if np.isfinite(eS).all():
            assert np.array_equal(S[i], S[i0]), k
            assert np.array_equal(h[i], h[i0] * 2.0 ** k), k
            assert np.array_equal(cal[i], cal[i0] * 2.0 ** k), k
            held += 1
        else:
            assert np.isnan(S[i]).all() and np.isnan(h[i]).all() and np.isnan(cal[i]).all(), k
    assert held >= 68 and -340 in ks and 330 in ks
    _hold('magnitude', 'k = 0', S[i0], h[i0], cal[i0], mag, seg)


def test_nonfinite_samples(eng):
    L = 300
    mag, seg = rotations(L=(L, L, L), seed=71)[:2]
    bad = []
    for v in (np.nan, np.inf, -np.inf):
        for s in range(3):
            for off in (0, 255, 256, L - 1):
                for c in (0, 2):
                    bad.append((v, seg[s][0] + off, c))
    good = [mag + 0.01 * k for k in range(4)]
    batch, kinds = [], []
    for i, (v, row, c) in enumerate(bad):
        m = mag.copy()
        m[row, c] = v
        batch.append(m)
        kinds.append(i)
        batch.append(good[i % 4])
        kinds.append(-1 - (i % 4))
    S, h, cal = _fed(eng, np.stack(batch), seg)
    Sg, hg, cg = _fed(eng, np.stack(good), seg)
    for j, k in enumerate(kinds):
        if k >= 0:
            assert np.isnan(S[j]).all() and np.isnan(h[j]).all() and np.isnan(cal[j]).all(), bad[k]
        else:
            g = -1 - k
            assert np.array_equal(S[j], Sg[g]) and np.array_equal(h[j], hg[g]) and np.array_equal(cal[j], cg[g])
    # at t, the first row of the x segment, in every sign
    assert any(row == seg[0][0] for _, row, _ in bad)
