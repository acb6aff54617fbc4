"""NumPy restatement of InsDataMgr.get_error_stats for sensor data (ins_data_manager.py:385-452, :524-541,
:717-808) on the b2ins noise spec, on top of oracle_np (gyro, accel) and mag_np (magnetometer).  Test
infrastructure only.

For a sensor x with truth ref, e = x - ref per run:
  * end-point statistics: max|e|, mean, std (ddof 0) over runs of e at the last row;
  * process statistics of run r: the same over the rows from a start index.
"""
import numpy as np

import oracle_np as onp
import mag_np

R2D = 180.0 / np.pi


def stats(x, ref, start):
    """x [R, m, C], ref [m, C] -> (end-point {'max','avg','std'} [C], process {'max','avg','std'} [R, C])."""
    e = np.asarray(x, dtype=np.float64) - np.asarray(ref, dtype=np.float64)[None]
    end = onp.array_stats(e[:, -1])
    es = e[:, start:]
    return end, {'max': np.max(np.abs(es), 1), 'avg': np.average(es, 1), 'std': np.std(es, 1)}


def imu(fs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_ids, vib_acc=None, vib_gyro=None):
    """gyro, accel [R, n, 3] of loop A on the b2ins stream (oracle_np.imu_noise)."""
    return onp.imu_noise(fs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_ids, vib_acc, vib_gyro)


def mag(ref_mag, mag_err, seed, run_ids):
    return mag_np.mag_gen(ref_mag, mag_err, mag_np.mag_normals(np.asarray(ref_mag).shape[0], run_ids, seed))


def gps(ref_gps, gps_err, gps_type, seed, run_ids):
    return onp.gps_gen(ref_gps, gps_err, gps_type, onp.gps_normals(np.asarray(ref_gps).shape[0], run_ids, seed))


def first_at(t, start_s):
    """The start row: the first time >= start_s, 0 past the end (ins_data_manager.py:774-782)."""
    idx = np.where(np.asarray(t) >= start_s)[0]
    return int(idx[0]) if idx.shape[0] else 0


def output_scale(units, out_units):
    """sim_data.convert_unit's factor per column (rad -> deg, rad/s -> deg/s)."""
    return np.array([R2D if (u, o) in (('rad', 'deg'), ('rad/s', 'deg/s')) else 1.0
                     for u, o in zip(units, out_units)])
