"""ORACLE (test infrastructure) -- the loosely-coupled filter spec (ekf_np.ins_loose) on SUPPLIED measurements.

ekf_np.ins_loose generates every run's IMU and GPS measurements from the truth and then filters them.  ins_loose
here runs that same spec with its generators handing back the supplied arrays instead (sensor_gen -> gyro /
accel, gps_gen -> gps), so there is one filter loop.  The initial state is ini plus, with ini_draw, the spec's
own initial-covariance draw; without it the draw is zero and goes through the same code.  The consistency
record needs the true biases, which supplied data do not have: it is not computed.  Without ref_nav there is no
end-point error.  On the generator's own measurements (with the draw) this is ekf_np.ins_loose bit for bit.
"""
import numpy as np

import ekf_np
import oracle_np as onp


class _FedOnp(object):
    """oracle_np as ekf_np.ins_loose sees it, with the measurement generators replaced by the supplied data; the
    normals it would draw for them are zeros (they feed only the unused bias truth), and so are the initial-state
    normals without ini_draw."""

    def __init__(self, gyro, accel, gps, ini_draw):
        self._meas = {'arw': gyro, 'vrw': accel}
        self._gps = gps
        self._draw = ini_draw

    def __getattr__(self, name):
        return getattr(onp, name)

    def noise_normals(self, n, run_ids, seed):
        z = np.zeros((np.asarray(run_ids).size, n, 3))
        return {'acc_gm': z, 'acc_w': z, 'gyr_gm': z, 'gyr_w': z}

    def gps_normals(self, m, run_ids, seed):
        return np.zeros((np.asarray(run_ids).size, m, 6))

    def sensor_gen(self, fs, ref, err, white_key, z_gm, z_w, vib=None):
        return self._meas[white_key]

    def gps_gen(self, ref_gps, gps_err, gps_type, z):
        return self._gps

    def normal_pair(self, t, pair, run, seed):
        # only ekf_np.initial_errors still draws here
        if self._draw:
            return onp.normal_pair(t, pair, run, seed)
        z = np.zeros(np.broadcast(np.asarray(t), np.asarray(run)).shape)
        return z, z


def ins_loose(fs, gyro, accel, gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err, ini, seed=0, run_ids=None,
              ini_draw=False, ref_nav=None, **kw):
    """The filter of ekf_np.ins_loose on gyro, accel [R, n, 3] and gps [R, m, 6] (LLA rad, m; NED m/s), GPS row j
    applied at IMU sample gps_idx[j] when gps_vis[j] > 0.  run_ids (default 0 .. R-1) name the initial draws
    (ini_draw).  ref_nav [n, 9] (optional): end_err.  kw: ini_att_std, earth_rot, want_hist, vel_rw, att_rw.
    Returns ekf_np.ins_loose's dict without the consistency entries (and without end_err if ref_nav is None)."""
    gyro, accel, gps = (np.asarray(a, dtype=np.float64) for a in (gyro, accel, gps))
    R, n, _ = gyro.shape
    run_ids = np.arange(R) if run_ids is None else np.asarray(run_ids)
    assert accel.shape == gyro.shape and gps.shape[0] == R and run_ids.size == R
    nav = np.zeros((n, 9)) if ref_nav is None else np.asarray(ref_nav, dtype=np.float64)
    saved = ekf_np.onp
    ekf_np.onp = _FedOnp(gyro, accel, gps, ini_draw)
    try:
        out = ekf_np.ins_loose(fs, np.zeros((n, 3)), np.zeros((n, 3)), nav, gps[0], gps_idx, gps_vis, gyro_err,
                               accel_err, gps_err, seed, run_ids, ini, stats_start=n, **kw)
    finally:
        ekf_np.onp = saved
    for k in ('nees', 'inside3', 'epochs'):
        del out[k]
    if ref_nav is None:
        del out['end_err']
    return out
