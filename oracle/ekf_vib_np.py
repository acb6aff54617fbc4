"""ORACLE (test infrastructure) -- the loosely-coupled filter spec (ekf_np.ins_loose) on vibrating sensors.

ekf_np.ins_loose draws its IMU through oracle_np.sensor_gen without a vibration term.  ins_loose here runs
that same spec with sensor_gen adding each sensor's vibration last (oracle_np.sensor_gen's `vib`): the
vibration oracle_np.imu_noise adds for the same runs (random: the PAIR_VIB normals; sinusoidal: zero phase
on the accelerometer, the PAIR_PHASE uniforms on the gyro) or, for the PSD model, a given per-run series
tiled to n as K5's consumers read it.  So the filter sees oracle_np's measurements of those runs.  Without
vibration it is ekf_np.ins_loose itself, unchanged.
"""
import numpy as np

import ekf_np
import oracle_np as onp


def vibration(fs, n, run_ids, seed, vib, sensor):
    """[R, n, 3] vibration of one sensor (0 accelerometer, 1 gyro) for the runs, or None.
    vib: None; a dict as oracle_np.imu_noise takes it (type 'random' | 'sinusoidal', x, y, z[, freq]); or
    the PSD model's series [R, 3, L] (time_series_from_psd's period), sample k reading column k % L."""
    if vib is None:
        return None
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    if not isinstance(vib, dict):
        s = np.asarray(vib, dtype=np.float64)
        assert s.ndim == 3 and s.shape[:2] == (run_ids.size, 3), s.shape
        return np.transpose(s[:, :, np.arange(n) % s.shape[2]], (0, 2, 1))
    amp = np.array([vib['x'], vib['y'], vib['z']], dtype=np.float64)
    if vib['type'] == 'random':
        z = onp.vib_normals(n, run_ids, seed)[sensor]
        return z * amp
    if vib['type'] == 'sinusoidal':
        phase = onp.gyro_vib_phase_uniforms(run_ids, seed) if sensor == 1 else None
        return onp.sinusoidal_vib(fs, n, amp, vib['freq'], phase)
    raise ValueError('unknown vibration type %r' % vib['type'])


class _VibratingOnp(object):
    """oracle_np as ekf_np.ins_loose sees it, with sensor_gen adding the vibration of its sensor last; it
    keeps what it made (by white-noise key: 'vrw' accelerometer, 'arw' gyro)."""

    def __init__(self, vib):
        self._vib = vib
        self.made = {}

    def __getattr__(self, name):
        return getattr(onp, name)

    def sensor_gen(self, fs, ref, err, white_key, z_gm, z_w):
        out = onp.sensor_gen(fs, ref, err, white_key, z_gm, z_w, self._vib[white_key])
        self.made[white_key] = out
        return out


def ins_loose(fs, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err,
              seed, run_ids, ini, vib_acc=None, vib_gyro=None, want_imu=False, **kw):
    """ekf_np.ins_loose (same arguments; kw: ini_att_std, earth_rot, stats_start, want_hist, vel_rw, att_rw)
    on measurements that carry vib_acc / vib_gyro (see vibration()).  want_imu: the output also holds the
    measurements the filter saw, 'gyro' and 'accel' [R, n, 3]."""
    n = ref_gyro.shape[0]
    hook = _VibratingOnp({'vrw': vibration(fs, n, run_ids, seed, vib_acc, 0),
                          'arw': vibration(fs, n, run_ids, seed, vib_gyro, 1)})
    saved = ekf_np.onp
    ekf_np.onp = hook
    try:
        out = ekf_np.ins_loose(fs, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis, gyro_err, accel_err,
                               gps_err, seed, run_ids, ini, **kw)
    finally:
        ekf_np.onp = saved
    if want_imu:
        out['gyro'], out['accel'] = hook.made['arw'], hook.made['vrw']
    return out
