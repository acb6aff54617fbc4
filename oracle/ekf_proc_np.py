"""ORACLE (test infrastructure) -- per-run process-error statistics of the loosely-coupled filter.

The reference's ins_loose is a stub, so the spec is the filter spec (ekf_np.ins_loose, or ekf_vib_np.ins_loose
on vibrating sensors) followed by the reference's statistics of its histories from a start index
(ins_data_manager.py:454-553, :761-808): the attitude error wrapped to [-pi, pi], the position as LLA
differences or in NED / ECEF metres (proc_pos_np), the velocity as plain differences; max|e|, mean and std
(ddof 0) per run and column.
"""
import numpy as np

import ekf_np
import ekf_vib_np
import oracle_np as onp
import proc_pos_np

FRAMES = ('', 'ned', 'ecef')       # B2INS_POS_FRAME_LLA, _NED, _ECEF


def process_stats(att, pos, vel, ref_nav, start, pos_frame=''):
    """[R, 3, 9] max|e|, mean, std of the att / pos / vel histories [R, n, 3] against ref_nav [n, 9] over samples
    >= start; pos_frame '' (LLA differences), 'ned' or 'ecef' (metres)."""
    a = onp.process_error_stats(att, ref_nav[:, 0:3], start, angle=True)
    p = proc_pos_np.process_error_stats(pos, ref_nav[:, 3:6], start, pos_frame)
    v = onp.process_error_stats(vel, ref_nav[:, 6:9], start)
    return np.stack([np.concatenate([a[k], p[k], v[k]], axis=1) for k in ('max', 'avg', 'std')], axis=1)


def ins_loose(fs, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err, seed,
              run_ids, ini, proc_start, pos_frame='', vib_acc=None, vib_gyro=None, **kw):
    """The filter spec with its histories (kw: ekf_np.ins_loose's ini_att_std, earth_rot, stats_start, vel_rw,
    att_rw), plus 'proc_stats' [R, 3, 9] from sample proc_start in pos_frame.  With vib_acc / vib_gyro the
    filter runs on vibrating sensors (ekf_vib_np.ins_loose)."""
    if vib_acc is None and vib_gyro is None:
        out = ekf_np.ins_loose(fs, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis, gyro_err, accel_err,
                               gps_err, seed, run_ids, ini, want_hist=True, **kw)
    else:
        out = ekf_vib_np.ins_loose(fs, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis, gyro_err,
                                   accel_err, gps_err, seed, run_ids, ini, vib_acc=vib_acc, vib_gyro=vib_gyro,
                                   want_hist=True, **kw)
    out['proc_stats'] = process_stats(out['att'], out['pos'], out['vel'], ref_nav, proc_start, pos_frame)
    return out
