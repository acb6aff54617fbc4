"""The self-initialising loosely-coupled filter (InsLoose(align_yaw=...)) on the CPU: the spec
(oracle/ekf_align_np.py) against the reference's levelling formulas, the fix-row rule, the P0 formulas, the NaN
rows, the host checks, and the end-point errors of a cold start against the truth-initialised filter."""
import math

import numpy as np
import pytest

from conftest import load_golden
import ekf_align_np
import ekf_np

FS = 100.0
DEMO_IMU = {'gyro_b': np.zeros(3), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
            'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
            'accel_b': np.zeros(3), 'accel_vrw': np.array([0.03119, 0.03009, 0.04779]),
            'accel_b_stability': np.array([4.29e-5, 5.72e-5, 8.02e-5]),
            'accel_b_corr': np.array([200.0, 200.0, 200.0])}       # demo_ins_loose.py:28-37


def _imu():
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True)


def _turn():
    """The 90-degree turn (true yaw 315 deg, 10 m/s) with its 10 Hz GPS truth; the first second is invisible."""
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    g = dict(load_golden('gps_90deg_rf0.npz'))
    g['gps_visibility'] = (g['gps_time'] >= 1.0).astype(np.float64)
    nav = np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1)
    return t, g, nav, np.rint(g['gps_time'] * FS).astype(np.int64)


@pytest.mark.parametrize('pitch,roll', [(0.0, 0.0), (0.1, -0.2), (-0.35, 0.6), (0.7, 2.5), (-1.2, -2.9)])
def test_levelling_recovers_static_tilts(pitch, roll):
    """Noise-free specific force of a static tilt, f_b = C(n->b) [0, 0, -g] with the reference's formulas
    (ins_loose.py:83-91: pitch = asin(a_x / |a|), roll = atan2(-a_y / |a|, -a_z / |a|))."""
    import oracle_np as onp
    c = onp.euler2dcm_zyx(np.array([[0.3, pitch, roll]]))[0]
    f = c.dot([0.0, 0.0, -9.79])
    accel = np.tile(f, (2, 12, 1))
    p, r = ekf_align_np.level(accel)
    assert np.abs(p - pitch).max() < 1e-12 and np.abs(r - roll).max() < 1e-12


def test_fix_row_rule():
    idx = np.array([0, 5, 9, 10, 20])
    assert ekf_align_np.fix_row(idx, [1, 1, 1, 1, 1]) == 2              # the latest at or before sample 9
    assert ekf_align_np.fix_row(idx, [1, 1, 0, 1, 1]) == 1              # invisible rows are skipped
    assert ekf_align_np.fix_row(idx, [0, 0, 0, 0, 1]) == 4              # none before: the first visible after
    assert ekf_align_np.fix_row(idx, [0, 0, 0, 0, 0]) is None
    assert ekf_align_np.start_sample(idx, 1) == 9 and ekf_align_np.start_sample(idx, 4) == 20
    _, g, _, gi = _turn()
    j = ekf_align_np.fix_row(gi, g['gps_visibility'])
    assert g['gps_visibility'][j] > 0 and not np.any(g['gps_visibility'][:j] > 0) and gi[j] > 9


def test_engine_fix_rule_is_the_spec_rule():
    from gnss_ins_sim_b200 import engine
    rng = np.random.default_rng(3)
    for _ in range(50):
        idx = np.sort(rng.choice(40, 8, replace=False))
        vis = (rng.random(8) > 0.5).astype(float)
        j = ekf_align_np.fix_row(idx, vis)
        assert engine.align_fix(idx, vis) == ((None, None) if j is None else (j, ekf_align_np.start_sample(idx, j)))


def test_host_checks():
    from gnss_ins_sim_b200.ins_loose import InsLoose
    with pytest.raises(ValueError):
        InsLoose(ini_pos_vel_att=np.zeros(9), align_yaw=0.1)
    with pytest.raises(ValueError):
        InsLoose(align_yaw='north')
    a = InsLoose(align_yaw='gps')
    idx, vel = np.array([0, 10, 20]), np.array([[0.5, 0.5], [3.0, 4.0], [3.0, 4.0]])
    with pytest.raises(ValueError):
        a.check_alignment(9, idx, np.ones(3), vel)                         # shorter than N
    with pytest.raises(ValueError):
        a.check_alignment(100, idx, np.zeros(3), vel)                      # no visible row
    with pytest.raises(ValueError):
        a.check_alignment(100, idx, np.ones(3), vel)                       # 0.71 m/s at the fix row
    assert a.check_alignment(100, idx, [0, 1, 1], vel) == 10
    assert InsLoose(align_yaw=0.2).check_alignment(100, idx, np.ones(3), vel) == 9    # speed is not needed
    with pytest.raises(ValueError):
        ekf_align_np.check(100, idx, np.ones(3), 'gps', vel)


def test_p0_and_nan_rows():
    """P0 entries are the formulas of DESIGN.md section 11; histories are NaN before the state exists."""
    t, g, nav, gi = _turn()
    imu = _imu()
    o = ekf_align_np.ins_loose_gen(FS, t['ref_gyro'][:300], t['ref_accel'][:300], nav[:300], g['ref_gps'][:30],
                                   gi[:30], g['gps_visibility'][:30], imu.gyro_err, imu.accel_err, imu.gps_err, 7,
                                   np.arange(4), 'gps', want_hist=True, want_imu=True)
    s0 = o['start']
    assert s0 == gi[o['fix_row']] and s0 > 9
    gap = (s0 - 9) / FS
    ae, ge, ge_s = imu.accel_err, imu.gyro_err, imu.gps_err
    sv = np.broadcast_to(np.asarray(ge_s['stdv'], dtype=float), (3,))
    v = o['gps'][:, o['fix_row'], 3:5]
    for r in range(4):
        p0 = o['p0'][r]
        assert np.allclose(p0[0:3], np.asarray(ge_s['stdp']) ** 2, rtol=1e-15)
        assert np.allclose(p0[3:6], sv ** 2, rtol=1e-15)
        for c, ax in ((0, 1), (1, 0)):           # N from accelerometer y (roll), E from x (pitch)
            lev = (ae['b'][ax] ** 2 + ae['b_drift'][ax] ** 2 + ae['vrw'][ax] ** 2 * FS / 10) / 9.80665 ** 2
            grow = ge['arw'][c] ** 2 * gap + (ge['b'][c] ** 2 + ge['b_drift'][c] ** 2) * gap ** 2
            assert p0[6 + c] == pytest.approx(lev + grow, rel=1e-14)
        yv = (sv[0] ** 2 * v[r, 1] ** 2 + sv[1] ** 2 * v[r, 0] ** 2) / (v[r, 0] ** 2 + v[r, 1] ** 2) ** 2
        grow = ge['arw'][2] ** 2 * gap + (ge['b'][2] ** 2 + ge['b_drift'][2] ** 2) * gap ** 2
        assert p0[8] == pytest.approx(yv + grow, rel=1e-14)
        assert np.array_equal(p0[9:], ekf_np.default_p0(ge, ae, ge_s, (0.02, 0.005, 0.005))[9:])
    assert np.all(np.isnan(o['att'][:, :9])) and not np.any(np.isnan(o['att'][:, 9:]))
    for k in ('pos', 'vel'):
        assert np.all(np.isnan(o[k][:, :s0])) and not np.any(np.isnan(o[k][:, s0:]))
    assert np.all(o['wb'][:, :s0] == 0.0) and np.all(o['ab'][:, :s0] == 0.0)
    assert np.array_equal(o['pos'][:, s0], o['gps'][:, o['fix_row'], 0:3])
    assert np.allclose(wrap(o['att'][:, 9, 0] - np.arctan2(v[:, 1], v[:, 0])), 0.0, atol=1e-15)
    # the fed form on the generator's own measurements is the generated form
    f = ekf_align_np.ins_loose(FS, o['gyro'], o['accel'], o['gps'], gi[:30], g['gps_visibility'][:30],
                               imu.gyro_err, imu.accel_err, imu.gps_err, 'gps', want_hist=True)
    assert np.array_equal(f['pos'], o['pos'], equal_nan=True) and np.array_equal(f['end_bias'], o['end_bias'])


def wrap(x):
    return (np.asarray(x) + math.pi) % (2 * math.pi) - math.pi


def test_cold_start_end_errors_near_the_truth_initialised_filter():
    """The 90-degree turn with 'gps' heading over 64 runs: the RMS end-point position error (N, E metres) of the
    cold start stays within a factor 1.5 of the truth-initialised filter's.  (Spec run: 0.78 and 0.78 m.)"""
    t, g, nav, gi = _turn()
    imu = _imu()
    runs = np.arange(64)
    a = ekf_align_np.ins_loose_gen(FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], gi, g['gps_visibility'],
                                   imu.gyro_err, imu.accel_err, imu.gps_err, 11, runs, 'gps')
    b = ekf_np.ins_loose(FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], gi, g['gps_visibility'],
                         imu.gyro_err, imu.accel_err, imu.gps_err, 11, runs, t['ini'])

    def rms_m(e):
        import oracle_np as onp
        rm, rn, _, _, cl = onp.geo_param(nav[-1, 3], nav[-1, 5])
        return np.sqrt(np.mean((e[:, 3] * rm) ** 2 + (e[:, 4] * rn * cl) ** 2))
    ra, rb = rms_m(a['end_err']), rms_m(b['end_err'])
    print('aligned %.3f m, truth-initialised %.3f m' % (ra, rb))
    assert np.all(np.isfinite(a['end_err']))
    assert ra < 1.5 * rb
    assert np.abs(wrap(a['end_err'][:, 0])).max() < 0.1


def test_filter_loop_is_ekf_np():
    """The aligned spec's filter loop (ekf_align_np.filter_from), started at sample 0 from ekf_np.ins_loose's initial
    state (truth + the P0 draw) on the same measurements, is ekf_np.ins_loose bit for bit: histories, end state,
    bias estimates and the consistency record.  So the two specs cannot drift apart."""
    import oracle_np as onp
    t, g, nav, gi = _turn()
    imu = _imu()
    ge, ae, gs = imu.gyro_err, imu.accel_err, imu.gps_err
    n, runs, seed = 400, np.arange(3, 8), 9
    ref = ekf_np.ins_loose(FS, t['ref_gyro'][:n], t['ref_accel'][:n], nav[:n], g['ref_gps'][:40], gi[:40],
                           g['gps_visibility'][:40], ge, ae, gs, seed, runs, t['ini'], stats_start=50, want_hist=True,
                           vel_rw=0.02)
    # ekf_np.ins_loose's measurements, bias truth and initial state, restated from its own helpers
    z = onp.noise_normals(n, runs, seed)
    accel = onp.sensor_gen(FS, t['ref_accel'][:n], ae, 'vrw', z['acc_gm'], z['acc_w'])
    gyro = onp.sensor_gen(FS, t['ref_gyro'][:n], ge, 'arw', z['gyr_gm'], z['gyr_w'])
    bias_g = np.asarray(ge['b'])[None, None] + onp.bias_drift(ge['b_corr'], ge['b_drift'], n, FS, z['gyr_gm'])
    bias_a = np.asarray(ae['b'])[None, None] + onp.bias_drift(ae['b_corr'], ae['b_drift'], n, FS, z['acc_gm'])
    gps = onp.gps_gen(g['ref_gps'][:40], gs, 0, onp.gps_normals(40, runs, seed))
    p0 = ekf_np.default_p0(ge, ae, gs, (0.02, 0.005, 0.005))
    e0 = ekf_np.initial_errors(runs, seed, p0)
    ini, R = t['ini'], runs.size
    c_t = onp.euler2dcm_zyx(np.tile(ini[6:9], (R, 1)))
    rm, rn, _, _, cl = onp.geo_param(ini[0], ini[2])
    pos = np.tile(ini[0:3], (R, 1))
    pos[:, 0] += e0[:, 0] / (rm + ini[2])
    pos[:, 1] += e0[:, 1] / ((rn + ini[2]) * cl)
    pos[:, 2] -= e0[:, 2]
    vel = onp._mtv(c_t, np.tile(ini[3:6], (R, 1))) + e0[:, 3:6]
    att = ekf_np.dcm2euler_zyx(np.einsum('rij,rjk->rik', c_t, np.eye(3)[None] + ekf_np.skew(e0[:, 6:9])))
    hist = {k: np.zeros((R, n, 3)) for k in ('att', 'pos', 'vel', 'wb', 'ab')}
    att, pos, vel, bg, ba, P, acc = ekf_align_np.filter_from(
        FS, gyro, accel, gps, gi[:40], g['gps_visibility'][:40], ge, ae, gs, 0, 0, att, pos, vel,
        np.tile(np.diag(p0), (R, 1, 1)), hist, True, nav[:n], bias_g, bias_a, 50, 0.02, 0.0)
    for k in hist:
        assert np.array_equal(hist[k], ref[k]), k
    assert np.array_equal(np.concatenate([bg, ba], 1), ref['end_bias'])
    assert np.array_equal(np.einsum('rii->ri', P), ref['P_diag_end'])
    assert acc['cnt'] == ref['epochs'] and acc['cnt'] > 0
    assert np.array_equal(acc['nees'] / acc['cnt'], ref['nees'])
    assert np.array_equal(acc['inside'] / acc['cnt'], ref['inside3'])
