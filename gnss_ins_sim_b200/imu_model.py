"""IMU / GPS / odometer error profiles -- the parameter source of the hot path.

Mirrors gnss_ins_sim.sim.imu_model (imu_model.py:18-61 built-in profiles, :62-205
constructor, :207-352 setters): same constructor, attribute names, units and
exceptions, so an `IMU` made here drops into code written for the reference.

One deliberate difference (SURVEY 7, "quirks not to copy"): the reference hands out
references to module-level dicts and a dict-valued `accuracy` overwrites them in place,
so building a second IMU silently changes the first.  Here every IMU owns private copies.

Units (as in the reference after its conversions, imu_model.py:138-143):
  gyro  b, b_drift [rad/s], arw [rad/s/sqrt(Hz)], b_corr [s]
  accel b, b_drift [m/s^2], vrw [m/s^2/sqrt(Hz)], b_corr [s]
and, only where a dict accuracy gives them, the IEEE Std 952 terms the reference does not model (the columns Q, K
and R of Allan(fit=True)'s noise_gyro / noise_accel):
  gyro  q [rad], rrw [rad/s^2/sqrt(Hz)], rr [rad/s^2]
  accel q [m/s], rrw [m/s^3/sqrt(Hz)], rr [m/s^3]
and the run-to-run errors (1 sigma, drawn once per Monte-Carlo run; DESIGN.md section 4):
  gyro  b_std [rad/s], sf [-], ma [rad] (3x3, zero diagonal)
  accel b_std [m/s^2], sf [-], ma [rad] (3x3, zero diagonal)
"""
import math

import numpy as np

D2R = math.pi / 180

# grade -> (gyro bias instability [deg/h], gyro ARW [deg/sqrt(h)],
#           accel bias instability [m/s^2], accel VRW [m/s/sqrt(h)], mag noise std [uT])
# imu_model.py:18-25 (low, AHRS380), :30-37 (mid, IMU381), :44-51 (high, HG9900)
_GRADES = {
    'low-accuracy': (10.0, 0.75, 2.0e-4, 0.05, 0.1),
    'mid-accuracy': (3.5, 0.25, 5.0e-5, 0.03, 0.01),
    'high-accuracy': (0.1, 2.0e-3, 3.6e-6, 2.5e-5, 0.001),
}
_CORR_TIME = 100.0  # s, all built-in grades


def _three(v):
    return np.array([v, v, v], dtype=np.float64)


def gyro_profile(grade):
    drift, arw, _, _, _ = _GRADES[grade]
    return {'b': _three(0.0) * D2R, 'b_drift': _three(drift) * D2R / 3600.0,
            'b_corr': _three(_CORR_TIME), 'arw': _three(arw) * D2R / 60.0}


def accel_profile(grade):
    _, _, drift, vrw, _ = _GRADES[grade]
    return {'b': _three(0.0), 'b_drift': _three(drift), 'b_corr': _three(_CORR_TIME),
            'vrw': _three(vrw) / 60.0}


def mag_profile(grade):
    return {'si': np.eye(3), 'hi': _three(0.0), 'std': _three(_GRADES[grade][4])}


def gps_profile():
    """imu_model.py:53-55"""
    return {'stdp': np.array([5.0, 5.0, 7.0]), 'stdv': np.array([0.05, 0.05, 0.05])}


def odo_profile():
    """imu_model.py:58-60"""
    return {'scale': 0.99, 'stdv': 0.1}


_REQUIRED = ('gyro_b', 'gyro_b_stability', 'gyro_arw', 'accel_b', 'accel_b_stability', 'accel_vrw')
# optional IEEE Std 952 terms: accuracy key -> (stored key, factor from the datasheet unit to SI)
_TERMS = {
    'gyro': {'gyro_q': ('q', D2R),                       # deg -> rad
             'gyro_rrw': ('rrw', D2R / 3600.0 / 60.0),    # deg/h/sqrt(h) -> rad/s^2/sqrt(Hz)
             'gyro_rr': ('rr', D2R / 3600.0 / 3600.0)},   # deg/h^2 -> rad/s^2
    'accel': {'accel_q': ('q', 1.0),                     # m/s
              'accel_rrw': ('rrw', 1.0 / 60.0),          # m/s^2/sqrt(h) -> m/s^3/sqrt(Hz)
              'accel_rr': ('rr', 1.0 / 3600.0)},         # m/s^2/h -> m/s^3
}
_TERM_KEYS = ('q', 'rrw', 'rr')
# optional run-to-run errors (1 sigma): accuracy key -> (stored key, factor from the datasheet unit to SI)
_RUN_ERRS = {
    'gyro': {'gyro_b_std': ('b_std', D2R / 3600.0),       # deg/h -> rad/s
             'gyro_sf': ('sf', 1e-6),                     # ppm
             'gyro_ma': ('ma', D2R)},                     # deg -> rad
    'accel': {'accel_b_std': ('b_std', 1.0),             # m/s^2
              'accel_sf': ('sf', 1e-6),                   # ppm
              'accel_ma': ('ma', D2R)},                   # deg -> rad
}
_RUN_ERR_KEYS = ('b_std', 'sf', 'ma')


def _terms(accuracy, sensor):
    """The IEEE Std 952 terms of one sensor an accuracy dict gives, in SI units (absent keys are not stored)."""
    out = {}
    for key, (stored, scale) in _TERMS[sensor].items():
        if key in accuracy:
            v = np.broadcast_to(np.array(accuracy[key], dtype=np.float64), (3,)) * scale
            if not np.all(np.isfinite(v)) or (stored != 'rr' and np.any(v < 0.0)):
                raise ValueError('%s must be finite%s' % (key, '' if stored == 'rr' else ' and >= 0'))
            out[stored] = v
    return out


def _run_err_value(key, stored, value):
    """One run-to-run error in SI units, checked: b_std and sf [3], ma 3x3 (a scalar is every off-diagonal) with a
    zero diagonal; every value finite and >= 0."""
    v = np.array(value, dtype=np.float64)
    if stored == 'ma':
        v = v * (1.0 - np.eye(3)) if v.ndim == 0 else v.reshape(3, 3)
        if np.any(np.diag(v) != 0.0):
            raise ValueError('%s must have a zero diagonal' % key)
    else:
        v = np.broadcast_to(v, (3,)).copy()
    if not np.all(np.isfinite(v)) or np.any(v < 0.0):
        raise ValueError('%s must be finite and >= 0' % key)
    return v


def _run_errs(accuracy, sensor):
    """The run-to-run errors of one sensor an accuracy dict gives, in SI units (absent keys are not stored)."""
    return {stored: _run_err_value(key, stored, np.array(accuracy[key], dtype=np.float64) * scale)
            for key, (stored, scale) in _RUN_ERRS[sensor].items() if key in accuracy}


class IMU(object):
    """IMU error model; see the module docstring.  accuracy: 'low-accuracy' |
    'mid-accuracy' | 'high-accuracy' | dict with gyro_b [deg/h], gyro_arw [deg/sqrt(h)],
    gyro_b_stability [deg/h], accel_b [m/s^2], accel_vrw [m/s/sqrt(h)],
    accel_b_stability [m/s^2] and optionally gyro_b_corr / accel_b_corr [s] (missing ->
    inf -> white bias drift), mag_si, mag_hi, mag_std, and the IEEE Std 952 terms gyro_q [deg],
    gyro_rrw [deg/h/sqrt(h)], gyro_rr [deg/h^2], accel_q [m/s], accel_rrw [m/s^2/sqrt(h)],
    accel_rr [m/s^2/h] (missing -> zero; stored as gyro_err / accel_err 'q', 'rrw', 'rr' in SI units), and the
    run-to-run errors (1 sigma) gyro_b_std [deg/h], accel_b_std [m/s^2], gyro_sf / accel_sf [ppm], gyro_ma /
    accel_ma [deg] (a scalar for every off-diagonal, or 3x3 with a zero diagonal) (missing -> zero; stored as
    'b_std', 'sf', 'ma' in SI units)."""

    def __init__(self, accuracy='low-accuracy', axis=6, gps=True, gps_opt=None,
                 odo=False, odo_opt=None):
        if axis == 9:
            self.magnetometer = True
        elif axis == 6:
            self.magnetometer = False
        else:
            raise ValueError('axis should be either 6 or 9.')

        if isinstance(accuracy, str):
            if accuracy not in _GRADES:
                raise ValueError('accuracy is not a valid string.')
            self.gyro_err = gyro_profile(accuracy)
            self.accel_err = accel_profile(accuracy)
            self.mag_err = mag_profile(accuracy)
        elif isinstance(accuracy, dict):
            if not all(k in accuracy for k in _REQUIRED):
                raise ValueError('accuracy should at least have keys: \n' +
                                 'gyro_b, gyro_b_stability, gyro_arw, ' +
                                 'accel_b, accel_b_stability and accel_vrw')
            inf3 = _three(float('inf'))
            as_arr = lambda v: np.array(v, dtype=np.float64)  # noqa: E731
            self.gyro_err = {
                'b': as_arr(accuracy['gyro_b']) * D2R / 3600.0,
                'b_drift': as_arr(accuracy['gyro_b_stability']) * D2R / 3600.0,
                'b_corr': as_arr(accuracy['gyro_b_corr']) if 'gyro_b_corr' in accuracy else inf3,
                'arw': as_arr(accuracy['gyro_arw']) * D2R / 60.0}
            self.accel_err = {
                'b': as_arr(accuracy['accel_b']),
                'b_drift': as_arr(accuracy['accel_b_stability']),
                'b_corr': as_arr(accuracy['accel_b_corr']) if 'accel_b_corr' in accuracy
                else inf3.copy(),
                'vrw': as_arr(accuracy['accel_vrw']) / 60.0}
            self.gyro_err.update(_terms(accuracy, 'gyro'))
            self.accel_err.update(_terms(accuracy, 'accel'))
            self.gyro_err.update(_run_errs(accuracy, 'gyro'))
            self.accel_err.update(_run_errs(accuracy, 'accel'))
            self.mag_err = mag_profile('low-accuracy')
            if self.magnetometer:
                if 'mag_std' not in accuracy:
                    raise ValueError('Magnetometer is enabled, ' +
                                     'but its noise std is not specified.')
                self.mag_err['std'] = as_arr(accuracy['mag_std'])
            self.mag_err['si'] = as_arr(accuracy['mag_si']) if 'mag_si' in accuracy else np.eye(3)
            self.mag_err['hi'] = as_arr(accuracy['mag_hi']) if 'mag_hi' in accuracy \
                else _three(0.0)
        else:
            raise TypeError('accuracy is not valid.')

        self.gps = bool(gps)
        self.gps_err = None
        if self.gps:
            self.gps_err = self._opt(gps_opt, ('stdp', 'stdv'), gps_profile(),
                                     'gps_opt should have key: stdp and stdv',
                                     'gps_opt should be None or a dict')
        self.odo = bool(odo)
        self.odo_err = None
        if self.odo:
            self.odo_err = self._opt(odo_opt, ('scale', 'stdv'), odo_profile(),
                                     'odo_opt should have key: scale and stdv',
                                     'odo_opt should be None or a dict')

    @staticmethod
    def _opt(opt, keys, default, msg_keys, msg_type):
        if opt is None:
            return default
        if not isinstance(opt, dict):
            raise TypeError(msg_type)
        if not all(k in opt for k in keys):
            raise ValueError(msg_keys)
        return opt

    @staticmethod
    def _set(current, value, profiles, what):
        if isinstance(value, str):
            if value not in _GRADES:
                raise ValueError('%s is not a valid string.' % what)
            return profiles(value)
        if isinstance(value, dict):
            for k in value:
                if k not in current and k not in _TERM_KEYS and k not in _RUN_ERR_KEYS:
                    raise ValueError('unsupported key: %s in %s' % (k, what))
                current[k] = _run_err_value(k, k, value[k]) if k in _RUN_ERR_KEYS else value[k]
            return current
        raise TypeError('%s is not valid.' % what)

    def set_gyro_error(self, gyro_error='low-accuracy'):
        """imu_model.py:207-236: grade string, or dict of {'b','arw','b_drift','b_corr'}
        IN THE STORED (SI) UNITS, exactly as the reference assigns them, and of 'q', 'rrw', 'rr'
        (Allan(fit=True)'s Q, K and R of a gyro axis: columns 0, 3 and 4 of noise_gyro), and of the run-to-run
        errors 'b_std' [rad/s], 'sf' [-], 'ma' [rad] (checked as IMU(accuracy=dict) checks them)."""
        self.gyro_err = self._set(self.gyro_err, gyro_error, gyro_profile, 'gyro_error')

    def set_accel_error(self, accel_error='low-accuracy'):
        """imu_model.py:238-267; also 'q', 'rrw', 'rr' as for set_gyro_error (noise_accel's columns), and
        'b_std' [m/s^2], 'sf', 'ma'."""
        self.accel_err = self._set(self.accel_err, accel_error, accel_profile, 'accel_error')

    def set_mag_error(self, mag_error='low-accuracy'):
        """imu_model.py:321-352 (no-op without a magnetometer)"""
        if self.magnetometer:
            self.mag_err = self._set(self.mag_err, mag_error, mag_profile, 'mag_error')

    def set_gps(self, gps_error=None):
        """imu_model.py:269-290"""
        if self.gps:
            self.gps_err = self._opt(gps_error, ('stdp', 'stdv'), gps_profile(),
                                     'gps_error should have key: stdp and stdv',
                                     'gps_error should be None or a dict')

    def set_odo(self, odo_error=None):
        """imu_model.py:292-313.  (The reference checks for 'stdp' here, a typo that makes
        every dict fail; this checks the keys the odometer model actually has.)"""
        if self.odo:
            self.odo_err = self._opt(odo_error, ('scale', 'stdv'), odo_profile(),
                                     'odo_error should have key: scale and stdv',
                                     'odo_error should be None or a dict')
