"""The reference's process-error statistics of LLA positions in metres (get_error_stats('pos',
err_stats_start >= 0, extra_opt='ned' | 'ecef') in ref_frame 0), restated in NumPy on top of oracle_np.
Test infrastructure."""
import numpy as np

import oracle_np as onp


def ecef_to_ned(lat, lon):
    """attitude.ecef_to_ned, attitude.py:596-603: rot_y(-pi/2 - lat) . rot_z(lon), vectorised over
    lat, lon [...] -> [..., 3, 3] (rot_y, rot_z: attitude.py:617-663)."""
    a = -onp.HALF_PI - np.asarray(lat, dtype=np.float64)
    sa, ca = np.sin(a), np.cos(a)
    so, co = np.sin(lon), np.cos(lon)
    z, o = np.zeros_like(sa), np.ones_like(sa)
    ry = np.stack([np.stack([ca, z, -sa], -1), np.stack([z, o, z], -1), np.stack([sa, z, ca], -1)], -2)
    rz = np.stack([np.stack([co, so, z], -1), np.stack([-so, co, z], -1), np.stack([z, z, o], -1)], -2)
    return ry @ rz


def lla_array_error(x, r, pos_frame):
    """InsDataMgr.array_error lla == 1 ('ned') / 2 ('ecef') branch, ins_data_manager.py:543-552:
    lla2ecef(x) - lla2ecef(r), for 'ned' rotated by ecef_to_ned of each row of r.  x[..., n, 3], r[n, 3]."""
    err = onp.lla2ecef(x) - onp.lla2ecef(r)
    if pos_frame == 'ned':
        err = np.einsum('...ij,...j->...i', ecef_to_ned(r[..., 0], r[..., 1]), err)
    return err


def process_error_stats(x, ref, start_idx, pos_frame=''):
    """__process_error_stats (ins_data_manager.py:761-795) of LLA positions x[R,n,3] against ref[n,3] over
    samples >= start_idx -> dict of [R,3]: pos_frame 'ned' / 'ecef' in metres (calc_data_err with that
    extra_opt, :454-553), '' the LLA differences (oracle_np.process_error_stats)."""
    if pos_frame not in ('ned', 'ecef'):
        return onp.process_error_stats(x, ref, start_idx)
    err = lla_array_error(x[:, start_idx:], ref[None, start_idx:], pos_frame)
    return {'max': np.max(np.abs(err), 1), 'avg': np.average(err, 1), 'std': np.std(err, 1)}
