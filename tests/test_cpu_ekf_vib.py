"""The loosely-coupled filter spec on vibrating sensors (oracle/ekf_vib_np.py).

The spec's measurements are oracle_np's for the same runs, vibration included; without vibration the spec
is ekf_np.ins_loose bit for bit; and vibration the filter model does not know about makes it overconfident,
which raising vel_model_std / att_model_std by sigma sqrt(dt) (the InsLoose recipe) repairs."""
import math

import numpy as np
import pytest

from conftest import load_golden
import ekf_np
import ekf_vib_np
import oracle_np as onp

DEMO_IMU = {'gyro_b': np.zeros(3), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
            'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
            'accel_b': np.zeros(3), 'accel_vrw': np.array([0.03119, 0.03009, 0.04779]),
            'accel_b_stability': np.array([4.29e-5, 5.72e-5, 8.02e-5]),
            'accel_b_corr': np.array([200.0, 200.0, 200.0])}       # demo_ins_loose.py:28-37
FS = 100.0
# a PSD table up to fs / 2, in the (n, 4) form Sim takes as env
PSD = np.stack([np.linspace(0.0, 50.0, 26), np.full(26, 1e-4), np.linspace(1e-4, 4e-4, 26),
                np.full(26, 2e-4)], axis=1)


def _imu():
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True)


def _env(text):
    from gnss_ins_sim_b200.sim import parse_env
    return parse_env(text, FS)


def _turn_case(n=None):
    """The 90-degree-turn trajectory in ref_frame 0 with its 10 Hz GPS truth, cut to n samples."""
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    g = dict(load_golden('gps_90deg_rf0.npz'))
    g['gps_visibility'] = np.ones_like(g['gps_visibility'])
    nav = np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1)
    idx = np.rint(g['gps_time'] * 100.0).astype(np.int64)
    n = n or t['ref_gyro'].shape[0]
    keep = idx < n
    return (t['ref_gyro'][:n], t['ref_accel'][:n], nav[:n], g['ref_gps'][keep], idx[keep],
            g['gps_visibility'][keep], t['ini'])


def _psd_series(n, run_ids, seed, sensor):
    """time_series_from_psd of every run and axis on the PSD phase normals: [R, 3, n]."""
    v = _env(PSD)
    L = min(n + n % 2, 16384) // 2 + 1             # the N // 2 + 1 phases time_series_from_psd reads
    z = onp.psd_phase_normals(L, run_ids, seed, sensor)
    return np.stack([np.stack([onp.time_series_from_psd(v[ax], v['freq'], FS, n, z[r, c])[1]
                               for c, ax in enumerate('xyz')]) for r in range(len(run_ids))])


@pytest.mark.parametrize('kind', ['random', 'sinusoidal', 'psd', 'random_acc_sinusoidal_gyro'])
def test_spec_measurements_are_oracle_np_imu(kind):
    rg, ra, nav, gps, idx, vis, ini = _turn_case(300)
    imu, seed, runs = _imu(), 7, np.arange(5, 9)
    n = rg.shape[0]
    if kind == 'psd':
        va, vg = _psd_series(n, runs, seed, 0), _psd_series(n, runs, seed, 1)
    elif kind == 'random_acc_sinusoidal_gyro':
        va, vg = _env('[0.05 0.02 0.03]g-random'), _env('[0.5 0.2 0.3]d-7.5Hz-sinusoidal')
    else:
        tail = '-random' if kind == 'random' else '-7.5Hz-sinusoidal'
        va, vg = _env('[0.05 0.02 0.03]g' + tail), _env('[0.5 0.2 0.3]d' + tail)
    o = ekf_vib_np.ins_loose(FS, rg, ra, nav, gps, idx, vis, imu.gyro_err, imu.accel_err, imu.gps_err, seed,
                             runs, ini, vib_acc=va, vib_gyro=vg, want_imu=True)
    if kind == 'psd':
        z = onp.noise_normals(n, runs, seed)
        ref_a = onp.sensor_gen(FS, ra, imu.accel_err, 'vrw', z['acc_gm'], z['acc_w'], np.transpose(va, (0, 2, 1)))
        ref_g = onp.sensor_gen(FS, rg, imu.gyro_err, 'arw', z['gyr_gm'], z['gyr_w'], np.transpose(vg, (0, 2, 1)))
    else:
        ref_g, ref_a = onp.imu_noise(FS, rg, ra, imu.gyro_err, imu.accel_err, seed, runs, vib_acc=va, vib_gyro=vg)
    assert np.array_equal(o['accel'], ref_a) and np.array_equal(o['gyro'], ref_g)
    quiet_g, quiet_a = onp.imu_noise(FS, rg, ra, imu.gyro_err, imu.accel_err, seed, runs)
    assert not np.array_equal(o['accel'], quiet_a) and not np.array_equal(o['gyro'], quiet_g)


def test_psd_series_is_tiled_as_time_series_from_psd():
    """A series of period N = 16384 read at k % N is time_series_from_psd's output for n > N."""
    v, runs, seed, n = _env(PSD), np.arange(2), 3, 20000
    z = onp.psd_phase_normals(8193, runs, seed, 0)
    period = np.stack([np.stack([onp.time_series_from_psd(v[ax], v['freq'], FS, 16384, z[r, c])[1]
                                 for c, ax in enumerate('xyz')]) for r in range(2)])
    long = np.stack([np.stack([onp.time_series_from_psd(v[ax], v['freq'], FS, n, z[r, c])[1]
                               for c, ax in enumerate('xyz')]) for r in range(2)])
    assert np.array_equal(ekf_vib_np.vibration(FS, n, runs, seed, period, 0), np.transpose(long, (0, 2, 1)))


def test_no_vibration_is_the_spec():
    rg, ra, nav, gps, idx, vis, ini = _turn_case(400)
    imu = _imu()
    args = (FS, rg, ra, nav, gps, idx, vis, imu.gyro_err, imu.accel_err, imu.gps_err, 2025, np.arange(5, 11), ini)
    a = ekf_np.ins_loose(*args, stats_start=100, want_hist=True, vel_rw=0.02)
    b = ekf_vib_np.ins_loose(*args, stats_start=100, want_hist=True, vel_rw=0.02, vib_acc=None, vib_gyro=None)
    assert sorted(a) == sorted(b)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_vibration_needs_the_model_noise_recipe():
    """64 runs of the 90-degree turn, seed 11, statistics from sample 100, random vibration of 0.05 g on the
    accelerometer and 0.5 deg/s on the gyro: the default model is overconfident in velocity and attitude;
    vel_model_std = sqrt(0.02^2 + sa^2 dt), att_model_std = sg sqrt(dt) makes it consistent again."""
    rg, ra, nav, gps, idx, vis, ini = _turn_case()
    imu = _imu()
    va, vg = _env('[0.05 0.05 0.05]g-random'), _env('[0.5 0.5 0.5]d-random')
    dt = 1.0 / FS

    def run(**kw):
        o = ekf_vib_np.ins_loose(FS, rg, ra, nav, gps, idx, vis, imu.gyro_err, imu.accel_err, imu.gps_err, 11,
                                 np.arange(64), ini, stats_start=100, vib_acc=va, vib_gyro=vg, **kw)
        return o['nees'].mean(0), o['inside3'].mean(0).min()

    nees, inside = run(vel_rw=0.02)
    assert nees[1] > 6.0 and nees[2] > 6.0 and inside < 0.9, (nees, inside)
    nees, inside = run(vel_rw=math.sqrt(0.02 ** 2 + va['x'] ** 2 * dt), att_rw=vg['x'] * math.sqrt(dt))
    assert np.all(nees > 1.5) and np.all(nees < 5.0) and inside > 0.97, (nees, inside)
