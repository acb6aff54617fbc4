"""Logged-data directories: the reference Sim's file input (gnss_ins_sim/sim/ins_sim.py:415-451,
:508-559, :796-832 and sim_data.py:78-115, :187-260), restated.

A directory holds one .csv per data set: `<name>.csv` (e.g. time.csv, ref_pos.csv) or
`<name>-<key>.csv` for the key-th set of a per-run quantity (gyro-0.csv, accel-0.csv); the first
row names the columns and may give their units in brackets, `gyro_x (deg/s)`.  Values are
converted to the simulation's internal units (rad, rad/s, m, m/s, m/s^2, sec).
"""
import os

import numpy as np

D2R = np.pi / 180.0

# internal units of the data the engine understands (ins_data_manager.py:68-205)
INTERNAL_UNITS = {
    'time': ['sec'], 'gps_time': ['sec'], 'gps_visibility': [''],
    'ref_pos': ['rad', 'rad', 'm'], 'ref_vel': ['m/s'] * 3, 'ref_att_euler': ['rad'] * 3,
    'ref_att_quat': [''] * 4, 'ref_gyro': ['rad/s'] * 3, 'ref_accel': ['m/s^2'] * 3,
    'ref_gps': ['rad', 'rad', 'm', 'm/s', 'm/s', 'm/s'], 'ref_odo': ['m/s'], 'ref_mag': ['uT'] * 3,
    'gyro': ['rad/s'] * 3, 'accel': ['m/s^2'] * 3,
    'gps': ['rad', 'rad', 'm', 'm/s', 'm/s', 'm/s'], 'odo': ['m/s'], 'mag': ['uT'] * 3,
}


def name_and_key(file_name):
    """'accel-0.csv' -> ('accel', 0); 'ref_pos.csv' -> ('ref_pos', None); not a csv -> (None, None)
    (ins_sim.py:508-535)."""
    file_name = file_name.lower()
    if not file_name.endswith('.csv'):
        return None, None
    name, key = file_name[:-4], None
    i = name.rfind('-')
    if i != -1:
        key = name[i + 1:]
        name = name[:i]
        if key.isdigit():
            key = int(key)
    return name, key


def file_units(path):
    """Units in brackets in the header row, one per column, else None (ins_sim.py:537-559)."""
    with open(path) as fp:
        cols = fp.readline().split(',')
    units = []
    for c in cols:
        lo, hi = c.find('('), c.rfind(')')
        if lo != -1 and hi != -1 and hi > lo:
            units.append(c[lo + 1:hi])
    return units if len(units) == len(cols) else None


def unit_scale(src, dst):
    """Per-column factor from src to dst units (sim_data.py:208-233); unknown pairs are left."""
    table = {('deg', 'rad'): D2R, ('deg/s', 'rad/s'): D2R, ('deg/hr', 'rad/s'): D2R / 3600.0,
             ('rad', 'deg'): 1.0 / D2R, ('rad/s', 'deg/s'): 1.0 / D2R, ('rad/s', 'deg/hr'): 3600.0 / D2R}
    scale = np.ones(len(dst))
    for i, (s, d) in enumerate(zip(src, dst)):
        if s != d:
            if (s, d) in table:
                scale[i] = table[(s, d)]
            else:
                print('Cannot convert unit from %s in %s to %s.' % (s, src, d))
    return scale


def convert_units(data, src, dst):
    """sim_data.convert_unit for one array (a copy)."""
    if len(src) != len(dst):
        raise ValueError('Units are of different lengths.')
    x = np.array(data, dtype=np.float64, copy=True)
    scale = unit_scale(src, dst)
    if x.ndim == 2:
        for i in range(min(len(scale), x.shape[1])):
            if scale[i] != 1.0:
                x[:, i] *= scale[i]
    elif x.ndim == 1:
        x = x * (scale if x.shape[0] == len(scale) else scale[0])
    return x


def _lla2ecef(lla):
    re, e2 = 6378137.0, 6.6943799901413e-3
    sl, cl = np.sin(lla[:, 0]), np.cos(lla[:, 0])
    r = re / np.sqrt(1.0 - e2 * sl * sl)
    rho = (r + lla[:, 2]) * cl
    return np.stack([rho * np.cos(lla[:, 1]), rho * np.sin(lla[:, 1]),
                     (r * (1.0 - e2) + lla[:, 2]) * sl], axis=1)


def convert_pos(data, units, ref_frame):
    """Position files against the reference frame (ins_sim.py:796-832).  In the virtual inertial
    frame an LLA file becomes metres: ECEF relative to the first sample, rotated, plus the first
    ECEF position.  The reference takes the rotation from the first RELATIVE row (all zeros),
    i.e. ecef_to_ned(0, 0); that is kept so that the two Sims agree."""
    data = np.array(data, dtype=np.float64, copy=True)
    units = list(units) if units is not None else None
    if ref_frame == 1:
        if units == ['deg', 'deg', 'm']:
            units = ['rad', 'rad', 'm']
            data[:, 0:2] *= D2R
        if units == ['rad', 'rad', 'm']:
            units = ['m', 'm', 'm']
            ecef = _lla2ecef(data)
            ini = ecef[0].copy()
            c_ne = np.array([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [-1.0, 0.0, 0.0]])   # ecef_to_ned(0, 0)
            data = (ecef - ini).dot(c_ne.T) + ini
    elif units == ['m', 'm', 'm']:
        units = ['rad', 'rad', 'm']
        print('Unsupported position conversion from xyz to LLA.')
    return data, units


def read_data_dir(path, ref_frame):
    """{name: array | {key: array}} in internal units for every supported .csv in `path`."""
    out = {}
    for fn in sorted(os.listdir(path)):
        name, key = name_and_key(fn)
        if name not in INTERNAL_UNITS:
            continue
        full = os.path.join(path, fn)
        data = np.genfromtxt(full, delimiter=',', skip_header=1)
        units = file_units(full)
        dst = list(INTERNAL_UNITS[name])
        if name in ('ref_pos', 'pos'):
            data, units = convert_pos(data, units, ref_frame)
            if ref_frame == 1:
                dst = ['m', 'm', 'm']
        if units is not None and units != dst:
            data = convert_units(data, units, dst)
        data = np.ascontiguousarray(data, dtype=np.float64)
        if key is None:
            out[name] = data
        else:
            out.setdefault(name, {})[key] = data
    return out


# ---- writing: Sim_data.save_to_file (sim_data.py:117-165) -----------------------------------------
# name -> (column legends, internal units, units written to the file)
_ANG3, _DEG3 = ['rad'] * 3, ['deg'] * 3
_NOISE = ['Q', 'N', 'B', 'K', 'R', 'B_min']
_NOISE_GYRO = ['rad', 'rad/s/sqrt(Hz)', 'rad/s', 'rad/s^2/sqrt(Hz)', 'rad/s^2', 'rad/s']
_NOISE_ACCEL = ['m/s', 'm/s^2/sqrt(Hz)', 'm/s^2', 'm/s^3/sqrt(Hz)', 'm/s^3', 'm/s^2']
OUTPUT_FORMAT = {
    'time': (['time'], ['sec'], ['sec']),
    'gps_time': (['gps_time'], ['sec'], ['sec']),
    'gps_visibility': (['gps_visibility'], [''], ['']),
    'ref_pos': (['ref_pos_lat', 'ref_pos_lon', 'ref_pos_alt'], ['rad', 'rad', 'm'], ['deg', 'deg', 'm']),
    'ref_vel': (['ref_vel_x', 'ref_vel_y', 'ref_vel_z'], ['m/s'] * 3, ['m/s'] * 3),
    'ref_att_euler': (['ref_Yaw', 'ref_Pitch', 'ref_Roll'], _ANG3, _DEG3),
    'ref_att_quat': (['q0', 'q1', 'q2', 'q3'], [''] * 4, [''] * 4),
    'ref_gyro': (['ref_gyro_x', 'ref_gyro_y', 'ref_gyro_z'], ['rad/s'] * 3, ['deg/s'] * 3),
    'ref_accel': (['ref_accel_x', 'ref_accel_y', 'ref_accel_z'], ['m/s^2'] * 3, ['m/s^2'] * 3),
    'ref_gps': (['ref_gps_lat', 'ref_gps_lon', 'ref_gps_alt', 'ref_gps_vN', 'ref_gps_vE', 'ref_gps_vD'],
                ['rad', 'rad', 'm', 'm/s', 'm/s', 'm/s'], ['deg', 'deg', 'm', 'm/s', 'm/s', 'm/s']),
    'ref_odo': (['ref_odo'], ['m/s'], ['m/s']),
    'ref_mag': (['ref_mag_x', 'ref_mag_y', 'ref_mag_z'], ['uT'] * 3, ['uT'] * 3),
    'gyro': (['gyro_x', 'gyro_y', 'gyro_z'], ['rad/s'] * 3, ['deg/s'] * 3),
    'accel': (['accel_x', 'accel_y', 'accel_z'], ['m/s^2'] * 3, ['m/s^2'] * 3),
    'gps': (['gps_lat', 'gps_lon', 'gps_alt', 'gps_vN', 'gps_vE', 'gps_vD'],
            ['rad', 'rad', 'm', 'm/s', 'm/s', 'm/s'], ['deg', 'deg', 'm', 'm/s', 'm/s', 'm/s']),
    'odo': (['odo'], ['m/s'], ['m/s']),
    'mag': (['mag_x', 'mag_y', 'mag_z'], ['uT'] * 3, ['uT'] * 3),
    'algo_time': (['algo_time'], ['sec'], ['sec']),
    'pos': (['pos_lat', 'pos_lon', 'pos_alt'], ['rad', 'rad', 'm'], ['deg', 'deg', 'm']),
    'vel': (['vel_x', 'vel_y', 'vel_z'], ['m/s'] * 3, ['m/s'] * 3),
    'att_euler': (['Yaw', 'Pitch', 'Roll'], _ANG3, _DEG3),
    'att_quat': (['q0', 'q1', 'q2', 'q3'], [''] * 4, [''] * 4),
    'ad_gyro': (['AD_gyro_x', 'AD_gyro_y', 'AD_gyro_z'], ['rad/s'] * 3, ['deg/s'] * 3),
    'ad_accel': (['AD_accel_x', 'AD_accel_y', 'AD_accel_z'], ['m/s^2'] * 3, ['m/s^2'] * 3),
    'hd_gyro': (['HD_gyro_x', 'HD_gyro_y', 'HD_gyro_z'], ['rad/s'] * 3, ['deg/s'] * 3),
    'hd_accel': (['HD_accel_x', 'HD_accel_y', 'HD_accel_z'], ['m/s^2'] * 3, ['m/s^2'] * 3),
    'algo_freq': (['algo_freq'], ['Hz'], ['Hz']),
    'psd_accel': (['PSD_accel_x', 'PSD_accel_y', 'PSD_accel_z'], ['m^2/s^4/Hz'] * 3, ['m^2/s^4/Hz'] * 3),
    'psd_gyro': (['PSD_gyro_x', 'PSD_gyro_y', 'PSD_gyro_z'], ['rad^2/s^2/Hz'] * 3, ['rad^2/s^2/Hz'] * 3),
    # Allan(fit=True): one row per axis (x, y, z), the IEEE Std 952 terms in SI units, written as they are
    'noise_gyro': (_NOISE, _NOISE_GYRO, _NOISE_GYRO),
    'noise_accel': (_NOISE, _NOISE_ACCEL, _NOISE_ACCEL),
}


def output_format(name, ref_frame):
    legend, units, out_units = OUTPUT_FORMAT[name]
    if ref_frame == 1 and name in ('ref_pos', 'pos'):        # ins_data_manager.py:207-230
        legend = [name + '_' + c for c in 'xyz']
        units = out_units = ['m', 'm', 'm']
    if ref_frame == 1 and name in ('ref_gps', 'gps'):
        legend = [name + '_' + c for c in ('x', 'y', 'z', 'vx', 'vy', 'vz')]
        units = out_units = ['m', 'm', 'm', 'm/s', 'm/s', 'm/s']
    return legend, units, out_units


def write_data(path, name, data, ref_frame):
    """`<name>.csv` or one `<name>-<key>.csv` per set, header `legend (unit)` per column, values in
    the output units -- what the reference's results(data_dir) writes and its file input reads."""
    legend, units, out_units = output_format(name, ref_frame)
    header = ','.join('%s (%s)' % (l, u) if u else l for l, u in zip(legend, out_units))
    os.makedirs(path, exist_ok=True)
    written = []
    items = data.items() if hasattr(data, 'items') else [(None, data)]
    for key, arr in items:
        fn = os.path.join(path, name + ('.csv' if key is None else '-%s.csv' % str(key)))
        np.savetxt(fn, convert_units(np.asarray(arr), units, out_units), header=header, delimiter=',',
                   comments='')
        written.append(fn)
    return written
