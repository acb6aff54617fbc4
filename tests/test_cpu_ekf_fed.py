"""The loosely-coupled filter on supplied measurements, without a GPU: the fed spec (oracle/ekf_fed_np.py), the
GPS-time -> IMU-sample rule, the argument checks of b2ins_ins_loose_fed_f64 and the plugin's model check."""
import ctypes

import numpy as np
import pytest

from conftest import load_golden, wrap_pi
import ekf_fed_np
import ekf_np
import oracle_np as onp

DEMO_IMU = {'gyro_b': np.zeros(3), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
            'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
            'accel_b': np.zeros(3), 'accel_vrw': np.array([0.03119, 0.03009, 0.04779]),
            'accel_b_stability': np.array([4.29e-5, 5.72e-5, 8.02e-5]),
            'accel_b_corr': np.array([200.0, 200.0, 200.0])}       # demo_ins_loose.py:28-37
FS = 100.0


def _imu(gps=True):
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=gps)


def _turn_case(n=400):
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    g = load_golden('gps_90deg_rf0.npz')
    nav = np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1)[:n]
    m = int(np.sum(g['gps_time'] * FS < n))
    idx = np.rint(g['gps_time'][:m] * FS).astype(np.int64)
    return t, g['ref_gps'][:m], nav, idx, np.ones(m), n


def test_fed_spec_on_generated_measurements_is_the_spec():
    """The generator's own measurements, fed with the same initial draw, give ekf_np.ins_loose's results exactly."""
    t, ref_gps, nav, idx, vis, n = _turn_case()
    imu, seed, run_ids = _imu(), 77, np.arange(3, 8)
    vis[4:7] = 0.0
    o = ekf_np.ins_loose(FS, t['ref_gyro'][:n], t['ref_accel'][:n], nav, ref_gps, idx, vis, imu.gyro_err,
                         imu.accel_err, imu.gps_err, seed, run_ids, t['ini'], want_hist=True, vel_rw=0.02)
    z = onp.noise_normals(n, run_ids, seed)
    accel = onp.sensor_gen(FS, t['ref_accel'][:n], imu.accel_err, 'vrw', z['acc_gm'], z['acc_w'])
    gyro = onp.sensor_gen(FS, t['ref_gyro'][:n], imu.gyro_err, 'arw', z['gyr_gm'], z['gyr_w'])
    gps = onp.gps_gen(ref_gps, imu.gps_err, 0, onp.gps_normals(ref_gps.shape[0], run_ids, seed))
    f = ekf_fed_np.ins_loose(FS, gyro, accel, gps, idx, vis, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'],
                             seed=seed, run_ids=run_ids, ini_draw=True, ref_nav=nav, want_hist=True, vel_rw=0.02)
    for k in ('end_err', 'end_bias', 'P_diag_end', 'att', 'pos', 'vel', 'wb', 'ab'):
        assert np.array_equal(f[k], o[k]), k
    assert 'nees' not in f and 'inside3' not in f


def test_fed_spec_without_draw_starts_at_ini():
    t, ref_gps, nav, idx, vis, n = _turn_case(50)
    ref_gps, idx, vis = ref_gps[1:], idx[1:], vis[1:]          # no update before the first history row
    imu = _imu()
    gps = np.tile(ref_gps, (2, 1, 1))
    gyro, accel = np.tile(t['ref_gyro'][:n], (2, 1, 1)), np.tile(t['ref_accel'][:n], (2, 1, 1))
    f = ekf_fed_np.ins_loose(FS, gyro, accel, gps, idx, vis, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'],
                             seed=5, want_hist=True)
    assert 'end_err' not in f
    assert np.array_equal(f['pos'][:, 0], np.tile(t['ini'][0:3], (2, 1)))
    assert np.abs(wrap_pi(f['att'][:, 0] - t['ini'][6:9])).max() < 1e-15       # the DCM round trip: an ulp at most
    assert np.array_equal(f['wb'][:, 0], np.zeros((2, 3)))


def test_gps_time_maps_to_the_nearest_imu_sample():
    from gnss_ins_sim_b200.ins_loose import gps_sample_index
    t, g = load_golden('traj_90deg_turn_100hz_rf0.npz'), load_golden('gps_90deg_rf0.npz')
    assert np.array_equal(gps_sample_index(FS, t['time'], g['gps_time']), np.rint(g['gps_time'] * FS))
    # nearest sample; a tie goes to the earlier one; half a sample beyond either end still maps to the end
    got = gps_sample_index(4.0, np.arange(10) * 0.25, [-0.125, 0.375, 0.625, 1.1, 2.375])
    assert got.dtype == np.int64 and got.tolist() == [0, 1, 2, 4, 9]
    assert gps_sample_index(FS, t['time'], []).shape == (0,)


@pytest.mark.parametrize('gps_time,time,msg', [
    ([0.01, 0.2], np.arange(10) / FS, 'outside the IMU series'),
    ([-0.0051], np.arange(10) / FS, 'outside the IMU series'),
    ([np.nan], np.arange(10) / FS, 'outside the IMU series'),
    ([0.045], np.r_[np.arange(4), np.arange(6, 10)] / FS, 'more than half a sample'),
    ([0.01, 0.012], np.arange(10) / FS, 'land on IMU samples 1 and 1'),
    ([0.05, 0.03], np.arange(10) / FS, 'land on IMU samples 5 and 3'),
    ([0.01], np.zeros(3), 'strictly increasing'),
])
def test_gps_time_mapping_rejects(gps_time, time, msg):
    from gnss_ins_sim_b200.ins_loose import gps_sample_index
    with pytest.raises(ValueError, match=msg):
        gps_sample_index(FS, time, gps_time)


def _fed_call(lib, cfg, ini_draw=0, bufs=None):
    """b2ins_ins_loose_fed_f64 with stand-in addresses: every case below fails an argument check, so none of them
    is ever dereferenced."""
    b = dict(gyro=1, accel=1, gps=1, gps_idx=1, gps_vis=1, ref_nav=None, end_err=None, end_bias=None, att=None,
             pos=None, vel=None, wb=None, ab=None)
    b.update(bufs or {})
    p = [None if b[k] is None else ctypes.c_void_p(0x1000 * b[k]) for k in
         ('gyro', 'accel', 'gps', 'gps_idx', 'gps_vis', 'ref_nav', 'end_err', 'end_bias', 'att', 'pos', 'vel',
          'wb', 'ab')]
    return lib.b2ins_ins_loose_fed_f64(cfg if cfg is None else ctypes.byref(cfg), ini_draw, *p, None)


@pytest.mark.parametrize('case,msg', [
    ('no_cfg', 'cfg is null'),
    ('fs', 'fs must be positive'),
    ('ini_draw', 'ini_draw must be 0 or 1'),
    ('end_err_alone', 'end_err and ref_nav'),
    ('ref_nav_alone', 'end_err and ref_nav'),
    ('n', 'n must be < 2^32'),
    ('no_gyro', 'null buffer'),
    ('no_gps', 'm > 0 needs gps'),
    ('dump_runs', 'dump_runs out of range'),
    ('some_dumps', 'given together'),
    ('vel_rw', 'vel_rw and att_rw'),
])
def test_fed_entry_rejects_bad_arguments_before_device_work(case, msg):
    from gnss_ins_sim_b200 import _lib, engine
    imu = _imu()
    cfg = engine._ekf_config(FS, 100, 3, 10, 1, imu.gyro_err, imu.accel_err, imu.gps_err, np.zeros(9), 0,
                             (0.02, 0.005, 0.005), True, -1, 0, 1, 0.02, 0.0)
    lib = _lib.load()
    ini_draw, bufs = 0, {}
    if case == 'no_cfg':
        cfg = None
    elif case == 'fs':
        cfg.fs = 0.0
    elif case == 'ini_draw':
        ini_draw = 2
    elif case == 'end_err_alone':
        bufs = {'end_err': 2}
    elif case == 'ref_nav_alone':
        bufs = {'ref_nav': 2}
    elif case == 'n':
        cfg.n = 1 << 32
    elif case == 'no_gyro':
        bufs = {'gyro': None}
    elif case == 'no_gps':
        bufs = {'gps': None}
    elif case == 'dump_runs':
        cfg.dump_runs = 4
    elif case == 'some_dumps':
        cfg.dump_runs = 3
        bufs = {'att': 3, 'pos': 4}
    elif case == 'vel_rw':
        cfg.vel_rw = -1.0
    assert _fed_call(lib, cfg, ini_draw, bufs) == _lib.ERR_ARG
    assert msg in lib.b2ins_last_error().decode()


def test_ins_loose_without_a_model_raises_model_missing():
    from gnss_ins_sim_b200.ins_loose import InsLoose, ModelMissing
    assert issubclass(ModelMissing, ValueError) and issubclass(ModelMissing, NotImplementedError)
    t, ref_gps, nav, idx, vis, n = _turn_case(50)
    with pytest.raises(ModelMissing):
        InsLoose(t['ini']).run([FS, t['ref_gyro'][:n], t['ref_accel'][:n], t['time'][:n], idx / FS, ref_gps])
    with pytest.raises(ModelMissing):
        InsLoose(t['ini']).run_batch(FS, t['ref_gyro'][None, :n], t['ref_accel'][None, :n], t['time'][:n], idx / FS,
                                     ref_gps[None])
    with pytest.raises(ValueError, match='gps=True'):
        InsLoose(imu=_imu(gps=False))
