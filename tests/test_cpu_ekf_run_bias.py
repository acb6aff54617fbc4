"""The run-to-run turn-on bias in the loosely-coupled filter without a GPU: the spec (oracle/ekf_rb_np.py) with and
without a turn-on bias, its consistency, the C entry points' bindings and argument checks, and what Sim accepts
and refuses for InsLoose."""
import ctypes

import numpy as np
import pytest

import ekf_align_np
import ekf_fed_np
import ekf_np
import ekf_rb_np
import run_err_np
from test_ekf import DEMO_IMU, _turn_case

# gyro_b_std 100 deg/h and accel_b_std 0.02 m/s^2: each well above the demo IMU's drift (3.5 deg/h, <= 8e-5 m/s^2)
BIG = dict(DEMO_IMU, gyro_b_std=np.full(3, 100.0), accel_b_std=np.full(3, 0.02))
BASE = {'gyro_b': [0.0] * 3, 'gyro_b_stability': [1.0] * 3, 'gyro_arw': [0.1] * 3, 'gyro_b_corr': [100.0] * 3,
        'accel_b': [0.0] * 3, 'accel_b_stability': [1e-4] * 3, 'accel_vrw': [0.05] * 3, 'accel_b_corr': [100.0] * 3}


def _imu(acc):
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy=acc, axis=6, gps=True)


def _spec(imu, runs=64, seed=11, **kw):
    t, g, nav, idx = _turn_case()
    return ekf_rb_np.ins_loose(100.0, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                            imu.gyro_err, imu.accel_err, imu.gps_err, seed, np.arange(runs), t['ini'],
                            stats_start=100, **kw)


def test_zero_turn_on_bias_is_the_spec_without_one():
    """Without b_std, or with a zero one, the spec is ekf_np's and ekf_align_np's, bit for bit: the draws are
    skipped and P0 gains + 0.0."""
    imu = _imu(DEMO_IMU)
    t, g, nav, idx = _turn_case()
    ref = ekf_np.ins_loose(100.0, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                           imu.gyro_err, imu.accel_err, imu.gps_err, 11, np.arange(6), t['ini'], stats_start=100,
                           want_hist=True)
    ge, ae = dict(imu.gyro_err, b_std=np.zeros(3)), dict(imu.accel_err, b_std=np.zeros(3))
    for gyro_err, accel_err in ((imu.gyro_err, imu.accel_err), (ge, ae)):
        got = ekf_rb_np.ins_loose(100.0, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                                  gyro_err, accel_err, imu.gps_err, 11, np.arange(6), t['ini'], stats_start=100,
                                  want_hist=True)
        assert set(got) == set(ref) | {'end_bias_err'}
        for k in ref:
            assert np.array_equal(got[k], ref[k]), k
        assert np.array_equal(ekf_rb_np.default_p0(gyro_err, accel_err, imu.gps_err, (0.02, 0.005, 0.005)),
                              ekf_np.default_p0(imu.gyro_err, imu.accel_err, imu.gps_err, (0.02, 0.005, 0.005)))
        for gap in (0.0, 0.37):
            assert np.array_equal(ekf_rb_np.p0_aligned(100.0, gyro_err, accel_err, imu.gps_err, (0.02, 0.005, 0.005),
                                                       gap),
                                  ekf_align_np.p0_aligned(100.0, imu.gyro_err, imu.accel_err, imu.gps_err,
                                                          (0.02, 0.005, 0.005), gap))
    # the swapped model is restored after every call
    assert ekf_np.default_p0 is not ekf_rb_np.default_p0 and ekf_align_np.p0_aligned is not ekf_rb_np.p0_aligned


def test_turn_on_bias_is_the_run_error_draw_and_enters_p0():
    imu = _imu(BIG)
    ge, ae = imu.gyro_err, imu.accel_err
    runs = np.arange(3, 9)
    for err, sensor in ((ge, 1), (ae, 0)):
        b = ekf_rb_np.turn_on_bias(err, sensor, 7, runs)
        assert np.array_equal(b, err['b'] + run_err_np.table(err, sensor, 7, runs)[:, :, 3])
        assert np.all(b != err['b'])
    p0 = ekf_rb_np.default_p0(ge, ae, imu.gps_err, (0.02, 0.005, 0.005))
    assert np.array_equal(p0[9:12], ge['b_drift'] ** 2 + ge['b'] ** 2 + ge['b_std'] ** 2)
    assert np.array_equal(p0[12:15], ae['b_drift'] ** 2 + ae['b'] ** 2 + ae['b_std'] ** 2)
    lev = ekf_rb_np.p0_aligned(100.0, ge, ae, imu.gps_err, (0.02, 0.005, 0.005), 0.0)[0, 6:8]
    want = (ae['b'] ** 2 + ae['b_drift'] ** 2 + ae['b_std'] ** 2 + ae['vrw'] ** 2 * 100.0 / 10) / 9.80665 ** 2
    assert np.array_equal(lev, want[[1, 0]])


def test_generated_measurements_carry_the_bias_and_the_fed_spec_takes_b_std_into_p0():
    """The spec's measurements are oracle_np's with b + b_run as the constant bias; filtered as supplied data by
    the fed spec (b_std in P0 only) they give the generated run, bit for bit."""
    imu = _imu(BIG)
    t, g, nav, idx = _turn_case()
    gen = _spec(imu, runs=4, seed=3, want_hist=True)
    meas = ekf_np.onp.noise_normals(1000, np.arange(4), 3)
    b_g = ekf_rb_np.turn_on_bias(imu.gyro_err, 1, 3, np.arange(4))
    b_a = ekf_rb_np.turn_on_bias(imu.accel_err, 0, 3, np.arange(4))
    gyro = ekf_np.onp.sensor_gen(100.0, t['ref_gyro'], dict(imu.gyro_err, b=b_g[:, None]), 'arw', meas['gyr_gm'],
                                 meas['gyr_w'])
    accel = ekf_np.onp.sensor_gen(100.0, t['ref_accel'], dict(imu.accel_err, b=b_a[:, None]), 'vrw', meas['acc_gm'],
                                  meas['acc_w'])
    gps = ekf_np.onp.gps_gen(g['ref_gps'], imu.gps_err, 0, ekf_np.onp.gps_normals(g['ref_gps'].shape[0], np.arange(4), 3))
    fed = ekf_rb_np.ins_loose_fed(100.0, gyro, accel, gps, idx, g['gps_visibility'], imu.gyro_err, imu.accel_err,
                                  imu.gps_err, t['ini'], seed=3, run_ids=np.arange(4), ini_draw=True, ref_nav=nav,
                                  want_hist=True)
    for k in ('end_err', 'end_bias', 'P_diag_end', 'att', 'pos', 'vel', 'wb', 'ab'):
        assert np.array_equal(fed[k], gen[k]), k
    # the truth: end_bias_err is the estimate minus b + b_run + d at n-1
    d_g = ekf_np.onp.bias_drift(imu.gyro_err['b_corr'], imu.gyro_err['b_drift'], 1000, 100.0, meas['gyr_gm'])
    assert np.allclose(gen['end_bias_err'][:, 0:3], gen['end_bias'][:, 0:3] - (b_g + d_g[:, -1]), rtol=0, atol=1e-18)


def test_spec_with_a_turn_on_bias_is_a_consistent_filter():
    """test_ekf.test_spec_is_a_consistent_filter's bounds on the 90-degree turn with BIG turn-on biases; and a
    control whose P0 leaves b_std out (the biases still in the data) is measurably less consistent.

    Where the control's thresholds come from (seed 11, 64 runs, 90 epochs): the spec's bias states are inside
    3 sigma in >= 99.7 % of epochs per axis (gyro 0.997 / 1.0 / 1.0, accel 0.997 / 0.998 / 1.0) and its block
    NEES are 3.5 / 3.0 / 2.8.  The control's bias states are inside in at most 10.9 % (gyro) and 1.5 % (accel)
    of epochs, and its velocity and attitude NEES are 73 and 86.  So the control must stay below 50 % inside
    on every bias state and above NEES 10 on those two blocks, and the spec above 97 % and below NEES 5."""
    imu = _imu(BIG)
    out = _spec(imu)
    assert out['epochs'] == 90
    nees = out['nees'].mean(0)
    assert np.all(nees > 1.5) and np.all(nees < 5.0), nees
    inside = out['inside3'].mean(0)
    assert inside.min() > 0.97, inside
    e = out['end_err']
    sig = np.sqrt(out['P_diag_end'].mean(0))
    assert (e[:, 3] * 6.37e6).std() < 2.0 * sig[0] and sig[0] < 2.5
    # the estimates recover most of each run's bias: end_bias_err is well inside the prior spread on every axis
    spread = out['end_bias_err'].std(0) / np.concatenate([imu.gyro_err['b_std'], imu.accel_err['b_std']])
    assert np.all(spread < 0.9), spread

    ctl = _spec(imu, model_b_std=False)
    assert np.array_equal(ctl['end_bias_err'].shape, (64, 6))
    assert ctl['inside3'].mean(0)[9:15].max() < 0.5, ctl['inside3'].mean(0)
    assert np.all(ctl['nees'].mean(0)[1:3] > 10.0), ctl['nees'].mean(0)


def test_new_entry_points_are_bound():
    from gnss_ins_sim_b200 import _lib
    for nm in ('b2ins_ins_loose_rx_f64', 'b2ins_ins_loose_fed_rx_f64'):
        assert nm in _lib.SIGNATURES
        assert getattr(_lib.load(), nm).argtypes == _lib.SIGNATURES[nm][1]


def _run_err(**kw):
    from gnss_ins_sim_b200 import _lib
    e = _lib.RunErr()
    for k, v in kw.items():
        if k == 'ma':
            for i in range(3):
                for j in range(3):
                    e.ma[i][j] = v[i][j]
        else:
            for c in range(3):
                getattr(e, k)[c] = v[c]
    return e


def test_entry_points_refuse_what_the_filter_cannot_model():
    """Non-zero sf or ma, and a b that is negative or not finite, give B2INS_ERR_ARG from the run-error check, ahead
    of the buffer checks (every buffer here is NULL) and so before any CUDA call."""
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    cfg = _lib.EkfConfig()
    cfg.fs, cfg.n, cfg.runs, cfg.m = 100.0, 100, 8, 0
    off = [[0.0, 1e-3, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]]
    bad = [(_run_err(sf=[0.0, 1e-4, 0.0]), 'scale factor'), (_run_err(ma=off), 'misalignment'),
           (_run_err(b=[0.0, -1e-3, 0.0]), 'finite and >= 0'), (_run_err(b=[float('nan'), 0.0, 0.0]), 'finite and >= 0'),
           (_run_err(b=[0.0, 0.0, float('inf')]), 'finite and >= 0')]
    nul = [None] * 15
    for e, text in bad:
        for g, a in ((e, None), (None, e)):
            rc = lib.b2ins_ins_loose_rx_f64(ctypes.byref(cfg), None, None, None, -1, 0, *nul, g, a, None, None)
            assert rc == _lib.ERR_ARG and text in lib.b2ins_last_error().decode(), (text, rc)
            rc = lib.b2ins_ins_loose_fed_rx_f64(ctypes.byref(cfg), None, 0, *nul[:13], g, a, None)
            assert rc == _lib.ERR_ARG and text in lib.b2ins_last_error().decode(), (text, rc)
    # a valid turn-on bias passes the check and meets the buffer check next
    ok = _run_err(b=[1e-4, 2e-4, 0.0])
    assert lib.b2ins_ins_loose_rx_f64(ctypes.byref(cfg), None, None, None, -1, 0, *nul, ok, ok, None, None) == _lib.ERR_ARG
    assert lib.b2ins_last_error().decode() == 'null buffer'
    empty = _lib.EkfConfig()
    empty.fs = 100.0
    assert lib.b2ins_ins_loose_rx_f64(ctypes.byref(empty), None, None, None, -1, 0, *nul, ok, ok, None, None) == _lib.OK


def _sim(acc, algo):
    from gnss_ins_sim_b200.imu_model import IMU
    from gnss_ins_sim_b200.sim import Sim
    n = 8
    traj = {k: np.zeros((n, 3)) for k in ('ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    traj['ref_odo'] = np.zeros(n)
    return Sim(100.0, traj, imu=IMU(acc, odo=True), algorithm=algo)


def test_sim_accepts_a_turn_on_bias_for_ins_loose_only():
    """InsLoose passes the refusal with b_std (and then stops at its own input check: this IMU has no GPS); every
    other run-to-run or IEEE Std 952 error is refused, naming only those keys; the odometer plugin still refuses
    b_std."""
    from gnss_ins_sim_b200.ins_loose import InsLoose
    from gnss_ins_sim_b200.free_integration_odo import FreeIntegration as FreeIntegrationOdo
    acc = dict(BASE, gyro_b_std=[10.0] * 3, accel_b_std=[1e-3] * 3)
    with pytest.raises(ValueError, match='ins_loose needs IMU'):
        _sim(acc, InsLoose(np.zeros(9))).run(1)
    for extra, keys in ((dict(gyro_sf=[100.0] * 3), ['gyro sf']), (dict(accel_ma=0.01), ['accel ma']),
                        (dict(gyro_q=[1e-6] * 3), ['gyro q']), (dict(accel_rrw=[1e-4] * 3), ['accel rrw']),
                        (dict(gyro_rr=[1e-3] * 3), ['gyro rr'])):
        sim = _sim(dict(acc, **extra), InsLoose(np.zeros(9)))
        with pytest.raises(ValueError) as e:
            sim.run(1)
        assert str(e.value).endswith(repr(keys)), str(e.value)
        assert 'b_std' not in str(e.value)
        assert 'gyro' not in sim.data and 'accel' not in sim.data
    sim = _sim(acc, FreeIntegrationOdo(np.zeros(9)))
    with pytest.raises(ValueError, match='scale-factor') as e:
        sim.run(1)
    assert "'gyro b_std'" in str(e.value) and "'accel b_std'" in str(e.value)
