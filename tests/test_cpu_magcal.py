"""The magnetometer calibration's NumPy oracle (oracle/magcal_np.py) against the reference's MagCalibrate
(tests/golden/magcal.npz), and the MagCal plugin's host-side checks.  No GPU needed.

Both oracle forms hold every golden case to 1e-12 relative, and to 1e-9 where the hard iron is 10 to 100 x
the field (kind 1): there the reference's own 4x4 normal equations are ill conditioned (cond ~1e12 at 100 x),
and its answer differs from a better-conditioned fit in the tenth digit.  Hard iron is held relative to the field
magnitude it estimates (hard_iron[3]), the scale of its errors, and the field radius within what the
reference's cancellation leaves of it (radius_cancellation)."""
import os
import tempfile
from datetime import date

import numpy as np
import pytest

import mag_np
import magcal_np as mc
from conftest import GOLDEN, load_golden, assert_close

TOL = {0: 1e-12, 1: 1e-9}
REF_MAG_STRIDE, MAG_CAL_STRIDE = 200, 8     # the rows the golden keeps (oracle/gen_golden_magcal.py)
_INPUTS = {}


def _cases(g):
    """The synthetic cases, their samples rebuilt from the golden's recipes."""
    for i in range(int(g['syn_count'])):
        mag, seg, kind = mc.golden_synthetic(g, i)
        assert abs(np.nansum(mag) - g['syn%d_nansum' % i]) <= 16 * mc.QUANTUM, 'case %d rebuilt differently' % i
        yield i, mag, seg, kind, g['syn%d_soft_iron' % i], g['syn%d_hard_iron' % i]


def golden_inputs(g):
    """(ref_mag [n, 3], ref_gyro [n, 3], mag [R, n, 3]) of the golden's Sim runs: the trajectory from the path
    generator with the reference's WMM coefficients (held to the golden's kept ref_mag rows), mag from its
    normals."""
    if 'sim' not in _INPUTS:
        from test_cpu_mag import write_cof
        from gnss_ins_sim_b200.sim import trajectory_from_motion_def
        with tempfile.TemporaryDirectory() as d:
            cof = write_cof(load_golden('mag_90deg.npz'), os.path.join(d, 'w.COF'))
            t = trajectory_from_motion_def(float(g['fs']), os.path.join(GOLDEN, 'motion_def-mag_cal.csv'), 1,
                                           magnetometer=True, wmm_file=cof, wmm_date=date(*map(int, g['date'])))
        assert_close(t['ref_mag'][::REF_MAG_STRIDE], g['ref_mag_rows'], 1e-12, 1.0, 'ref_mag')
        n = t['ref_mag'].shape[0]
        err = {'si': g['mag_si'], 'hi': g['mag_hi'], 'std': g['mag_std']}
        mag = mag_np.mag_gen(t['ref_mag'], err, mag_np.mag_normals(n, g['run_ids'], int(g['seed'])))
        _INPUTS['sim'] = (t['ref_mag'], t['ref_gyro'], mag)
    return _INPUTS['sim']


@pytest.mark.parametrize('form', ['direct', 'moments'])
def test_oracle_matches_reference_library(form):
    g = load_golden('magcal.npz')
    kinds = set()
    for i, mag, seg, kind, si, hi in _cases(g):
        kinds.add(kind)
        S, h = (mc.calibrate_direct(mag, seg)[:2] if form == 'direct' else mc.calibrate_moments(mag, seg))
        if kind == 2:
            assert np.isnan(si).all() and np.isnan(S).all() and np.isnan(h).all(), i
            continue
        assert_close(S, si, TOL[kind], 1.0, 'case %d soft_iron' % i)
        assert_close(h[0:3], hi[0:3], TOL[kind], abs(hi[3]), 'case %d hard_iron' % i)
        assert_close(h[3], hi[3], TOL[kind] * radius_cancellation(hi), 1.0, 'case %d field radius' % i)
    assert kinds == {0, 1, 2}


def radius_cancellation(hi):
    """The reference's radius is sqrt(p3 + |p|^2) with p3 = r^2 - |p|^2: it loses a factor 1 + |p|^2 / r^2 of
    relative accuracy to the cancellation (1.5e4 at a hard iron 100 x the field)."""
    return 1.0 + hi[0:3].dot(hi[0:3]) / (hi[3] * hi[3])


@pytest.mark.parametrize('form', ['direct', 'moments'])
def test_oracle_matches_reference_sim(form):
    g = load_golden('magcal.npz')
    seg = g['segments']
    ref_mag, _, mag = golden_inputs(g)
    for r in range(len(g['run_ids'])):
        if form == 'direct':
            S, h, cal = mc.calibrate_direct(mag[r], seg)
        else:
            S, h = mc.calibrate_moments(mag[r], seg)
            cal = mc.apply(mag[r], seg, S, h)
        assert_close(cal[::MAG_CAL_STRIDE], g['mag_cal_rows'][r], 1e-12, 1.0, 'mag_cal run %d' % r)
        assert_close(S, g['soft_iron'][r], 1e-12, 1.0, 'soft_iron run %d' % r)
        assert_close(h, g['hard_iron'][r][0], 1e-12, 1.0, 'hard_iron run %d' % r)
        # the estimate recovers si^-1 up to a scale: the calibration error is small at this noise
        e = mc.calibration_error(S, h, g['mag_si'], g['mag_hi'], np.linalg.norm(ref_mag[0]))
        assert np.abs(e[0:9]).max() < 0.02 and np.abs(e[9:]).max() < 1.0, e


def test_motion_rotations_are_clean():
    """The golden's segments lie inside single-axis rotations of at least 360 degrees."""
    g = load_golden('magcal.npz')
    ref_gyro = golden_inputs(g)[1]
    for a, (lo, hi) in enumerate(g['segments']):
        w = ref_gyro[lo:hi]
        assert np.abs(np.delete(w, a, axis=1)).max() <= 1e-12
        assert (hi - lo) * np.abs(w[:, a]).min() / float(g['fs']) >= 2 * np.pi


def test_moments_form_is_shift_invariant_at_large_hard_iron():
    """The sphere fit in the shifted frame: a 100 x |b| hard iron is recovered as well as a small one."""
    rng = np.random.default_rng(4)
    b = np.array([20.0, -5.0, 42.0])
    si = np.eye(3) + 0.05 * rng.standard_normal((3, 3))
    for hi_mag in (10.0, 4700.0):
        hi = rng.standard_normal(3)
        hi *= hi_mag / np.linalg.norm(hi)
        rows = []
        for ax in range(3):
            ang = np.linspace(0.0, 2.2 * np.pi, 2000)
            c, s = np.cos(ang), np.sin(ang)
            i, j = [(1, 2), (2, 0), (0, 1)][ax]
            bb = np.tile(b, (ang.size, 1))
            bb[:, i], bb[:, j] = c * b[i] + s * b[j], -s * b[i] + c * b[j]
            rows.append((bb + hi).dot(si.T))
        mag = np.concatenate(rows)
        S, h = mc.calibrate_moments(mag, ((0, 2000), (2000, 4000), (4000, 6000)))
        e = mc.calibration_error(S, h, si, hi, np.linalg.norm(b))
        assert np.abs(e[0:9]).max() < 1e-5 and np.abs(e[9:12]).max() < 1e-5 * hi_mag, (hi_mag, e)


def test_solve_flags_singular_systems():
    assert np.isnan(mc.solve(np.array([[1.0, 2.0], [2.0, 4.0]]), np.ones(2))).all()
    assert np.isnan(mc.solve(np.array([[np.nan, 0.0], [0.0, 1.0]]), np.ones(2))).all()
    x = mc.solve(np.array([[0.0, 2.0], [3.0, 1.0]]), np.array([4.0, 5.0]))
    assert np.allclose(x, [1.0, 2.0], rtol=0, atol=1e-15)


@pytest.mark.parametrize('bad', [None, ((0, 10), (10, 20)), ((0, 10), (10, 20), (20, 22)), ((-1, 10), (10, 20), (20, 30)),
                                 ((0, 10.5), (10, 20), (20, 30)), 'abc', ((0, np.nan), (10, 20), (20, 30)),
                                 ((5, 4), (10, 20), (20, 30))])
def test_magcal_rejects_bad_segments(bad):
    from gnss_ins_sim_b200.mag_calibrate import MagCal
    with pytest.raises(ValueError):
        MagCal(segments=bad)


def test_magcal_checks_segments_against_the_data():
    from gnss_ins_sim_b200.mag_calibrate import MagCal, check_segments
    a = MagCal(segments=((0, 10), (10, 20), (20, 30)))
    assert a.input == ['mag'] and a.output == ['soft_iron', 'hard_iron', 'mag_cal']
    assert check_segments(a.segments, 30).tolist() == [[0, 10], [10, 20], [20, 30]]
    with pytest.raises(ValueError):
        check_segments(a.segments, 29)
    with pytest.raises(ValueError):
        a.run_batch(np.zeros((1, 29, 3)))


def test_six_axis_imu_is_refused():
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.mag_calibrate import MagCal
    from gnss_ins_sim_b200.sim import Sim
    imu = imu_model.IMU(accuracy='mid-accuracy', axis=6, gps=False)
    sim = Sim([100.0, 0.0, 0.0], os.path.join(GOLDEN, 'motion_def-mag_cal.csv'), ref_frame=1, imu=imu,
              algorithm=MagCal(segments=((343, 1900), (2243, 3800), (4143, 5700))))
    with pytest.raises(ValueError, match='axis=9'):
        sim.run(2)
