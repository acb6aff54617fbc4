"""The exact magnetometer calibration (oracle/magcal_exact.py) and its bound on K10's rounding, without a GPU.

  * the exact reference equals a 200-bit evaluation of the reference's own steps (magcal_exact.direct_mp:
    plane fits on m, ranges over every sample, the [2c, 1] sphere fit on c = S m) on small cases of ten kinds;
  * it holds the reference library's golden at test_cpu_magcal's tolerances;
  * K10's algorithm emulated in float64 (magcal_np.calibrate_moments(order='kernel')) stays within the bound over
    the conditioning grid the GPU tests use, and on its exact class;
  * the bound is not vacuous: with hard iron up to 10 x the field and plane fits of condition up to 1e4 it is
    below 1e-11 of |S|, so an error of 1e-10 fails;
  * the emulation scales with the samples bit for bit from 2^-340 to 2^330 (the sphere fit's equilibration).
The worst emulation error / bound is printed (pytest -s)."""
import numpy as np
import pytest

import magcal_exact as me
import magcal_np as mc
from conftest import load_golden, assert_close
from test_cpu_magcal import TOL, radius_cancellation

FIELD = 45.0
HARD = (0.0, 1.0, 10.0, 1e2, 1e3, 1e4)         # x the field's magnitude
COND = (1.0, 1e3, 1e6)                           # of the soft iron
NOISE = (0.0, 0.01, 0.3)                         # x the field's magnitude


def rotations(L=(400, 400, 400), hard=10.0 / FIELD, cond=1.0, noise=0.3 / FIELD, seed=0, sweep=2.2):
    """(mag [sum L, 3], segments): a 45 uT field rotated about x, y and z (sweep x pi rad, L[k] samples each),
    measured as si (b + hi) + noise, si of condition `cond` around I + 5 %, |hi| = hard x 45 uT, noise its
    standard deviation in units of 45 uT."""
    rng = np.random.default_rng(seed)
    b = np.array([20.0, -5.0, 41.0])
    b *= FIELD / np.linalg.norm(b)
    Q, _ = np.linalg.qr(np.eye(3) + 0.05 * rng.standard_normal((3, 3)))
    si = Q.dot(np.diag(np.geomspace(1.0, 1.0 / cond, 3))).dot(Q.T) * (1 + 0.05 * rng.standard_normal())
    si = si + 0.05 * rng.standard_normal((3, 3)) * (cond == 1.0)
    hi = rng.standard_normal(3)
    hi *= hard * FIELD / np.linalg.norm(hi)
    rows = []
    for ax, n in enumerate(L):
        ang = np.linspace(0.0, sweep * np.pi, n)
        c, s = np.cos(ang), np.sin(ang)
        i, j = [(1, 2), (2, 0), (0, 1)][ax]
        bb = np.tile(b, (n, 1))
        bb[:, i], bb[:, j] = c * b[i] + s * b[j], -s * b[i] + c * b[j]
        rows.append((bb + hi).dot(si.T) + noise * FIELD * rng.standard_normal((n, 3)))
    e = np.cumsum((0,) + tuple(L))
    return np.concatenate(rows), ((e[0], e[1]), (e[1], e[2]), (e[2], e[3])), si, hi, FIELD


def conditioning_cases():
    """(name, mag, segments, model) over the hard iron x soft iron grid, and the noise sweep."""
    for h in HARD:
        for c in COND:
            mag, seg, si, hi, b = rotations(hard=h, cond=c, seed=int(h) % 97 + int(np.log10(c)))
            yield 'hard %g cond %g' % (h, c), mag, seg, (si, hi, b)
    for nz in NOISE:
        mag, seg, si, hi, b = rotations(noise=nz, seed=11)
        yield 'noise %g' % nz, mag, seg, (si, hi, b)


def within(got, ex, bnd):
    """max |got - ex| / bnd (0 where both are 0); inf where got is not finite."""
    got, ex, bnd = (np.asarray(a, dtype=np.float64) for a in (got, ex, bnd))
    if not np.isfinite(got).all():
        return np.inf
    err = np.abs(got - ex)
    return float(np.max(np.where(err == 0, 0.0, err / np.where(bnd > 0, bnd, np.inf))))


def check_against_exact(S, h, r, what):
    """K10's (or the emulation's) S, hard against the exact result r on its class; the worst error / bound."""
    nan = np.isnan(S).all() and np.isnan(h).all()
    if r['cls'] == 'singular':
        assert nan, '%s: singular case not NaN' % what
        return 0.0
    if r['cls'] == 'band' and nan:
        return 0.0
    assert not nan, '%s: NaN on a regular case (pivot %.3g)' % (what, r['pivot'])
    w = max(within(S, r['soft_iron'], r['b_soft']), within(h, r['hard_iron'], r['b_hard']))
    assert w <= 1.0, '%s: error / bound %.3g' % (what, w)
    return w


SMALL = {
    'clean rotations': lambda: rotations(L=(40, 40, 40), noise=0.0)[:2],
    'noisy rotations': lambda: rotations(L=(40, 40, 40), seed=1)[:2],
    'hard iron 100 x': lambda: rotations(L=(40, 40, 40), hard=100.0, seed=2)[:2],
    'soft iron cond 1e3': lambda: rotations(L=(40, 40, 40), cond=1e3, seed=3)[:2],
    'scaled 2^200': lambda: (rotations(L=(40, 40, 40), seed=4)[0] * 2.0 ** 200, ((0, 40), (40, 80), (80, 120))),
    'scaled 2^-200': lambda: (rotations(L=(40, 40, 40), seed=4)[0] * 2.0 ** -200, ((0, 40), (40, 80), (80, 120))),
    'segments z y x': lambda: (rotations(L=(40, 40, 40), seed=5)[0][::-1].copy(), ((80, 120), (40, 80), (0, 40))),
    'overlapping': lambda: (rotations(L=(40, 40, 40), seed=6)[0], ((0, 60), (30, 90), (70, 120))),
    'three rows each': lambda: (rotations(L=(3, 3, 3), seed=7, sweep=0.5)[0], ((0, 3), (3, 6), (6, 9))),
    'random samples': lambda: (np.random.default_rng(8).standard_normal((50, 3)) * 40 + 3,
                               ((0, 20), (15, 35), (30, 50))),
}


@pytest.mark.parametrize('kind', sorted(SMALL))
def test_exact_matches_reference_steps_at_200_bits(kind):
    mag, seg = SMALL[kind]()
    r = me.calibrate(mag, seg, want_bound=False)
    S, h = me.direct_mp(mag, seg)
    S = np.array([[float(v) for v in row] for row in S])
    h = np.array([float(v) for v in h])
    assert r['cls'] != 'singular'
    # both are one rounding of the same real number, unless it sits within 2^-190 of a rounding boundary
    for got, ref in ((r['soft_iron'], S), (r['hard_iron'], h)):
        assert (np.abs(got - ref) <= np.spacing(np.abs(ref))).all(), (kind, got - ref)


def test_exact_matches_reference_library():
    g = load_golden('magcal.npz')
    for i in range(int(g['syn_count'])):
        mag, seg, kind = mc.golden_synthetic(g, i)
        r = me.calibrate(mag, seg, want_bound=False)
        si, hi = g['syn%d_soft_iron' % i], g['syn%d_hard_iron' % i]
        if kind == 2:
            assert r['cls'] == 'singular' and np.isnan(r['soft_iron']).all(), i
            continue
        assert_close(r['soft_iron'], si, TOL[kind], 1.0, 'case %d soft_iron' % i)
        assert_close(r['hard_iron'][0:3], hi[0:3], TOL[kind], abs(hi[3]), 'case %d hard_iron' % i)
        assert_close(r['hard_iron'][3], hi[3], TOL[kind] * radius_cancellation(hi), 1.0, 'case %d radius' % i)


def test_emulation_within_bound_over_the_grid():
    worst = (0.0, None)
    classes = set()
    for name, mag, seg, model in conditioning_cases():
        r = me.calibrate(mag, seg, want_cal=True, model=model)
        classes.add(r['cls'])
        S, h = mc.calibrate_moments(mag, seg, order='kernel')
        w = check_against_exact(S, h, r, name)
        if np.isfinite(S).all():
            w = max(w, within(mc.apply(mag, seg, S, h), r['mag_cal'].astype(np.float64), r['b_cal']))
            w = max(w, within(mc.calibration_error(S, h, *model), r['err'], r['b_err']))
            assert w <= 1.0, name
        worst = max(worst, (w, name), key=lambda z: z[0])
    assert 'regular' in classes
    print('\nemulated K10: worst error / bound %.3g (%s)' % worst)


def plane_cond(mag, seg):
    """The largest condition number of the three plane-fit systems M^T M."""
    return max(np.linalg.cond(mag[a:b].T.dot(mag[a:b])) for a, b in seg)


def test_bound_is_not_vacuous():
    held = 0
    for h in (0.0, 1.0, 3.0, 10.0):
        for c in (1.0, 3.0, 10.0):
            mag, seg, si, hi, b = rotations(hard=h, cond=c, seed=21)
            if plane_cond(mag, seg) > 1e4:
                continue
            r = me.calibrate(mag, seg)
            assert r['cls'] == 'regular'
            rel = r['b_soft'].max() / np.abs(r['soft_iron']).max()
            assert rel <= 1e-11, (h, c, rel)
            # an error of 1e-10 relative on S fails the bound
            assert (1e-10 * np.abs(r['soft_iron']).max() > r['b_soft']).all()
            held += 1
    assert held >= 5


def test_bound_grows_with_conditioning():
    rel = []
    for h in (1.0, 100.0, 1e4):
        mag, seg = rotations(hard=h, seed=22)[:2]
        r = me.calibrate(mag, seg)
        rel.append(r['b_soft'].max() / np.abs(r['soft_iron']).max())
    assert rel[0] < rel[1] < rel[2], rel


def test_emulation_scales_bit_for_bit():
    """The equilibrated sphere fit: every scaling is a power of two, so from 2^-340 to 2^330 the result scales
    with the samples exactly; past that the moments leave the range of float64 and the result is all NaN."""
    mag, seg = rotations(seed=23)[:2]
    S0, h0 = mc.calibrate_moments(mag, seg, order='kernel')
    for k in range(-370, 371, 10):
        S, h = mc.calibrate_moments(mag * 2.0 ** k, seg, order='kernel')
        if -340 <= k <= 330:
            assert np.array_equal(S, S0) and np.array_equal(h, h0 * 2.0 ** k), k
        elif not (np.array_equal(S, S0) and np.array_equal(h, h0 * 2.0 ** k)):
            assert np.isnan(S).all() and np.isnan(h).all(), k
    for k in (-370, 370):
        S, h = mc.calibrate_moments(mag * 2.0 ** k, seg, order='kernel')
        assert np.isnan(S).all() and np.isnan(h).all(), k
