"""True-trajectory generation on the host -- the interface of gnss_ins_sim.pathgen.pathgen
(`path_gen`, pathgen.py:26-329; `parse motion definition` as Sim.__parse_motion does,
ins_sim.py:578-640), computed by the C++ restatement in csrc/pathgen_host.h through the C ABI
(b2ins_path_gen_ex_host).  CPU only: this is the one stage the north star keeps off the GPU."""
import ctypes
import math
import os
from io import StringIO

import numpy as np

from . import _lib, geomag

D2R = math.pi / 180
HIGH_MOBILITY = np.array([1.0, 0.5, 2.0])   # m/s^2, rad/s^2, rad/s (ins_sim.py:25)


def path_gen(ini_pos_vel_att, motion_def, output_def, mobility, ref_frame=0, magnet=False,
             wmm_file=None, wmm_date=None):
    """pathgen.path_gen: same arguments and the same result dictionary
    ('status', 'imu' (n,7), 'nav' (n,10), 'gps' (m,8), 'odo' (n,5), 'mag' (n,4) or []).
    Unlike the reference it does not modify motion_def / output_def in place.
    magnet: the field is the World Magnetic Model at the initial position (geomag.field_ned) from
    wmm_file (default: the installed gnss_ins_sim's WMM.COF) on wmm_date (default: today)."""
    lib = _lib.load()
    ini = np.ascontiguousarray(ini_pos_vel_att, dtype=np.float64).reshape(-1)[:9].copy()
    geo_mag_n = np.array(geomag.field_ned(ini, ref_frame, wmm_file, wmm_date)) if magnet else None
    md = np.ascontiguousarray(motion_def, dtype=np.float64)
    if md.ndim != 2 or md.shape[1] < 9:
        raise ValueError('motion_def must be (segments, 9)')
    md = np.ascontiguousarray(md[:, :9])
    od = np.asarray(output_def, dtype=np.float64)
    if od.shape != (3, 2):
        raise ValueError('output_def should be of size 3x2.')
    mob = np.ascontiguousarray(mobility, dtype=np.float64)
    fs, osr = float(od[0, 1]), float(od[0, 0])
    if (md[:, 7] < 0).any():
        i = int(np.where(md[:, 7] < 0)[0][0])
        raise ValueError('Time duration of %s-th command has negative time duration: %s.' % (i, md[i, 7]))
    rows = lib.b2ins_path_rows(_lib.host_ptr(md), md.shape[0], fs)
    if rows <= 0:
        raise ValueError('Total time duration in the motion definition file must be above 0.')
    want_gps, want_odo = od[1, 0] == 1, od[2, 0] == 1
    imu = np.zeros((rows, 7))
    nav = np.zeros((rows, 10))
    gps = np.zeros((rows, 8)) if want_gps else None
    odo = np.zeros((rows, 5)) if want_odo else None
    mag = np.zeros((rows, 4)) if magnet else None
    n_gps = ctypes.c_int64(0)
    n = lib.b2ins_path_gen_ex_host(_lib.host_ptr(ini), _lib.host_ptr(md), md.shape[0], fs, osr,
                                   float(od[1, 1]) if want_gps else 0.0, float(od[2, 1]) if want_odo else 0.0,
                                   _lib.host_ptr(mob), int(ref_frame), rows, _lib.host_ptr(imu),
                                   _lib.host_ptr(nav), _lib.host_ptr(gps), ctypes.byref(n_gps),
                                   _lib.host_ptr(odo), _lib.host_ptr(geo_mag_n), _lib.host_ptr(mag))
    if n < 0:
        raise ValueError('path_gen failed (%d): %s' % (n, lib.b2ins_last_error().decode()))
    return {'status': True, 'imu': imu[:n], 'nav': nav[:n], 'mag': mag[:n] if magnet else [],
            'gps': gps[:n_gps.value] if want_gps else [], 'odo': odo[:n] if want_odo else []}


def parse_motion(motion_def):
    """Motion-definition csv path or string -> (ini_pos_vel_att [rad], motion_def rows [rad]),
    as Sim.__parse_motion (ins_sim.py:578-610)."""
    try:
        if os.path.isfile(motion_def):
            ini = np.genfromtxt(motion_def, delimiter=',', skip_header=1, max_rows=1)
            way = np.genfromtxt(motion_def, delimiter=',', skip_header=3)
        else:
            ini = np.genfromtxt(StringIO(motion_def), delimiter=',', skip_header=1, max_rows=1)
            way = np.genfromtxt(StringIO(motion_def), delimiter=',', skip_header=3)
        if way.ndim == 1:
            way = way.reshape((1, len(way)))
        ini = np.array(ini[:9], dtype=np.float64)
        cmd = np.array(way[:, :9], dtype=np.float64)
    except Exception:
        raise ValueError('motion definition file/string must have nine columns '
                         'and at least four rows (two header rows + at least two data rows).')
    ini[0:2] *= D2R
    ini[6:9] *= D2R
    cmd[:, 1:4] *= D2R
    cmd[np.isnan(cmd)] = 0.0
    return ini, cmd


def parse_mode(mode):
    """Sim.__parse_mode (ins_sim.py:612-640): a string selects the built-in mobility; an array is
    [max acceleration m/s^2, max angular acceleration deg/s^2, max angular rate deg/s]."""
    if mode is None or isinstance(mode, str):
        return HIGH_MOBILITY.copy()
    if isinstance(mode, np.ndarray):
        if mode.shape != (3,):
            raise TypeError('mode should be of size (3,)')
        out = np.array(mode, dtype=np.float64)
        out[1:3] *= D2R
        return out
    raise TypeError('mode should be a string or a numpy array of size (3,)')
