"""ctypes binding of csrc/libb2ins.so (include/b2ins.h).  No CPU fallback: if the
library is missing or a call fails, the product path raises."""
import ctypes
import os

import numpy as np

from . import build as _build

c_double_p = ctypes.POINTER(ctypes.c_double)
c_int64_p = ctypes.POINTER(ctypes.c_int64)

OK, ERR_ARG, ERR_CUDA, ERR_NODEV = 0, 1, 2, 3
LAYOUT_RUN_MAJOR, LAYOUT_TIME_MAJOR, LAYOUT_CHANNEL_MAJOR = 0, 1, 2
VIB_NONE, VIB_RANDOM, VIB_SINUSOIDAL, VIB_SERIES = 0, 1, 2, 3
POS_FRAME_LLA, POS_FRAME_NED, POS_FRAME_ECEF = 0, 1, 2
ALIGN_OFF, ALIGN_YAW, ALIGN_GPS = 0, 1, 2


class SensorErr(ctypes.Structure):
    _fields_ = [('b', ctypes.c_double * 3), ('b_drift', ctypes.c_double * 3),
                ('b_corr', ctypes.c_double * 3), ('rw', ctypes.c_double * 3)]


class NoiseTerms(ctypes.Structure):
    _fields_ = [('q', ctypes.c_double * 3), ('k', ctypes.c_double * 3), ('r', ctypes.c_double * 3)]


class Vib(ctypes.Structure):
    _fields_ = [('type', ctypes.c_int32), ('series_len', ctypes.c_int32),
                ('amp', ctypes.c_double * 3), ('freq', ctypes.c_double),
                ('series', ctypes.c_void_p)]


class McConfig(ctypes.Structure):
    _fields_ = [('ref_frame', ctypes.c_int32), ('earth_rot', ctypes.c_int32),
                ('fs', ctypes.c_double), ('n', ctypes.c_int64), ('runs', ctypes.c_int64),
                ('run_offset', ctypes.c_int64), ('ini_offset', ctypes.c_int64),
                ('seed', ctypes.c_uint64),
                ('gyro_err', SensorErr), ('accel_err', SensorErr),
                ('vib_gyro', Vib), ('vib_accel', Vib),
                ('ini_sets', ctypes.c_int32), ('ini_rows', ctypes.c_int32),
                ('lanes_per_run', ctypes.c_int32), ('stats_start', ctypes.c_int32),
                ('dump_runs', ctypes.c_int64),
                ('algo', ctypes.c_int32), ('dump_stride', ctypes.c_int32),
                ('odo_scale', ctypes.c_double), ('odo_stdv', ctypes.c_double),
                ('ref_odo', ctypes.c_void_p), ('dump_odo', ctypes.c_void_p),
                ('dump_quat', ctypes.c_void_p)]


class EkfConfig(ctypes.Structure):
    _fields_ = [('fs', ctypes.c_double), ('n', ctypes.c_int64), ('runs', ctypes.c_int64),
                ('run_offset', ctypes.c_int64), ('m', ctypes.c_int64), ('seed', ctypes.c_uint64),
                ('gyro_err', SensorErr), ('accel_err', SensorErr),
                ('gps_stdp', ctypes.c_double * 3), ('gps_stdv', ctypes.c_double * 3),
                ('ini', ctypes.c_double * 9), ('ini_att_std', ctypes.c_double * 3),
                ('stats_start', ctypes.c_int64), ('dump_runs', ctypes.c_int64),
                ('dump_stride', ctypes.c_int32), ('earth_rot', ctypes.c_int32),
                ('vel_rw', ctypes.c_double), ('att_rw', ctypes.c_double)]


class EkfAlign(ctypes.Structure):
    _fields_ = [('mode', ctypes.c_int32), ('reserved', ctypes.c_int32), ('yaw', ctypes.c_double),
                ('yaw_var', ctypes.c_double)]


class B2insError(RuntimeError):
    pass


_I, _L, _D, _P, _U64 = ctypes.c_int, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p, ctypes.c_uint64
_SE, _VB, _MC = ctypes.POINTER(SensorErr), ctypes.POINTER(Vib), ctypes.POINTER(McConfig)
_NT = ctypes.POINTER(NoiseTerms)

# name -> (restype, argtypes); every symbol include/b2ins.h declares
SIGNATURES = {
    'b2ins_version': (_I, []),
    'b2ins_last_error': (ctypes.c_char_p, []),
    'b2ins_device_count': (_I, []),
    'b2ins_allan_num_tau': (_I, [_L, _D, c_int64_p, _I]),
    'b2ins_free_integration_f64': (_I, [_I, _D, _L, _L, _P, _P, _I, _P, _I, _I, _L, _I, _P, _P, _P, _I, _P]),
    'b2ins_free_integration_odo_f64': (_I, [_I, _D, _L, _L, _P, _P, _I, _P, _I, _I, _L, _I, _P, _P, _P, _I, _P]),
    'b2ins_free_integration_f64_host': (_I, [_I, _D, _L, _L, _P, _P, _I, _P, _I, _I, _L, _I, _P, _P, _P, _I]),
    'b2ins_imu_noise_f64': (_I, [_D, _L, _L, _P, _P, _SE, _SE, _VB, _VB, _U64, _L, _I, _P, _P, _P, _P]),
    'b2ins_imu_noise_f64_host': (_I, [_D, _L, _L, _P, _P, _SE, _SE, _VB, _VB, _U64, _L, _I, _P, _P, _P]),
    'b2ins_imu_noise_ex_f64': (_I, [_D, _L, _L, _P, _P, _SE, _SE, _NT, _NT, _VB, _VB, _U64, _L, _I, _P, _P, _P, _P]),
    'b2ins_imu_noise_ex_f64_host': (_I, [_D, _L, _L, _P, _P, _SE, _SE, _NT, _NT, _VB, _VB, _U64, _L, _I, _P, _P, _P]),
    'b2ins_gps_noise_f64': (_I, [_L, _L, _P, _P, _P, _I, _U64, _L, _P, _P]),
    'b2ins_mag_noise_f64': (_I, [_L, _L, _P, _P, _P, _P, _U64, _L, _P, _P]),
    'b2ins_magcal_f64': (_I, [_L, _L, c_int64_p, _P, _P, _P, _P, _U64, _L, _P, _P, _P, _P]),
    'b2ins_magcal_fed_f64': (_I, [_L, _L, c_int64_p, _P, _L, _L, _P, _P, _P, _P]),
    'b2ins_magcal_fed_f64_host': (_I, [_L, _L, c_int64_p, _P, _L, _L, _P, _P, _P]),
    'b2ins_imu_err_stats_f64': (_I, [_D, _L, _L, _P, _P, _SE, _SE, _VB, _VB, _U64, _L, _L, _P, _P, _P]),
    'b2ins_imu_err_stats_ex_f64': (_I, [_D, _L, _L, _P, _P, _SE, _SE, _NT, _NT, _VB, _VB, _U64, _L, _L, _P, _P, _P]),
    'b2ins_proc_stats_f64': (_I, [_L, _L, _I, _P, _P, _L, _P, _P, _P]),
    'b2ins_mc_free_integration_f64': (_I, [_MC, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'b2ins_mc_free_integration_ex_f64': (_I, [_MC, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'b2ins_mc_free_integration_f64_host': (_I, [_MC, _P, _P, _P, _P, _P, _P]),
    'b2ins_mc_plan_create': (_I, [_L, _L, _I, _I, ctypes.POINTER(ctypes.c_void_p)]),
    'b2ins_mc_plan_run': (_I, [_P, _MC, _P, _P, _P, _P, _P, _P]),
    'b2ins_mc_plan_destroy': (_I, [_P]),
    'b2ins_mc_plan_err_device': (_P, [_P]),
    'b2ins_mc_plan_stream': (_P, [_P]),
    'b2ins_error_stats_workspace_bytes': (_L, [_I]),
    'b2ins_error_partial_f64': (_I, [_L, _I, _P, _P, _P, _P]),
    'b2ins_error_partial2_f64': (_I, [_L, _I, _P, _P, _P, _P, _P]),
    'b2ins_error_stats_f64': (_I, [_L, _I, _P, _P, _P, _P]),
    'b2ins_error_stats_exchange_f64': (_I, [_L, _I, _P, _I, _I, ctypes.POINTER(ctypes.c_uint64), _U64, _P, _P, _P]),
    'b2ins_allan_workspace_bytes': (_L, [_L, _L]),
    'b2ins_allan_f64': (_I, [_D, _L, _L, _P, _L, _L, _L, _P, _P, _P, _P]),
    'b2ins_allan_mc_f64': (_I, [_D, _L, _L, _P, _P, _SE, _SE, _U64, _L, _P, _P, _P, _P]),
    'b2ins_allan_f64_host': (_I, [_D, _L, _L, _P, _L, _L, _L, _P, _P]),
    'b2ins_oallan_workspace_bytes': (_L, [_L, _L]),
    'b2ins_oallan_f64': (_I, [_D, _L, _L, _P, _L, _L, _L, _P, _P, _P, _P]),
    'b2ins_oallan_f64_host': (_I, [_D, _L, _L, _P, _L, _L, _L, _P, _P]),
    'b2ins_ohadamard_f64': (_I, [_D, _L, _L, _P, _L, _L, _L, _P, _P, _P, _P]),
    'b2ins_ohadamard_f64_host': (_I, [_D, _L, _L, _P, _L, _L, _L, _P, _P]),
    'b2ins_allan_fit_f64': (_I, [_D, _L, _L, _P, _L, _L, _P, _P]),
    'b2ins_allan_fit_f64_host': (_I, [_D, _L, _L, _P, _L, _L, _P]),
    'b2ins_psd_series_len': (_I, [_L]),
    'b2ins_psd_workspace_bytes': (_L, [_L, _L]),
    'b2ins_psd_series_f64': (_I, [_D, _L, _L, _I, _I, _P, _P, _U64, _L, _P, _P, _P]),
    'b2ins_welch_workspace_bytes': (_L, [_L, _L, _L, _L]),
    'b2ins_welch_f64': (_I, [_D, _L, _L, _P, _L, _L, _L, _L, _L, _P, _P, _P, _P, _P]),
    'b2ins_welch_f64_host': (_I, [_D, _L, _L, _P, _L, _L, _L, _L, _L, _P, _P, _P]),
    'b2ins_path_rows': (_L, [_P, _L, _D]),
    'b2ins_path_gen_host': (_L, [_P, _P, _L, _D, _D, _D, _D, _P, _I, _L, _P, _P, _P, c_int64_p, _P]),
    'b2ins_path_gen_ex_host': (_L, [_P, _P, _L, _D, _D, _D, _D, _P, _I, _L, _P, _P, _P, c_int64_p, _P, _P, _P]),
    'b2ins_ins_loose_f64': (_I, [ctypes.POINTER(EkfConfig)] + [_P] * 15),
    'b2ins_ins_loose_ex_f64': (_I, [ctypes.POINTER(EkfConfig), _VB, _VB] + [_P] * 15),
    'b2ins_ins_loose_fed_f64': (_I, [ctypes.POINTER(EkfConfig), _I] + [_P] * 14),
    'b2ins_ins_loose_proc_f64': (_I, [ctypes.POINTER(EkfConfig), _VB, _VB, _L, _I] + [_P] * 16),
    'b2ins_ins_loose_align_f64': (_I, [ctypes.POINTER(EkfConfig), ctypes.POINTER(EkfAlign), _VB, _VB, _L, _I]
                                  + [_P] * 16),
    'b2ins_ins_loose_fed_align_f64': (_I, [ctypes.POINTER(EkfConfig), ctypes.POINTER(EkfAlign)] + [_P] * 14),
    'b2ins_diag_dfma_rate': (_I, [c_double_p]),
    'b2ins_diag_auto_lanes': (_I, [_L, _I, _I]),
    'b2ins_diag_mc_shape': (_I, [_I, _I, ctypes.POINTER(ctypes.c_int)]),
    'b2ins_diag_psd_plan': (_I, [_L, ctypes.POINTER(ctypes.c_int)]),
    'b2ins_diag_noise_plan': (_I, [_D, _L, _L, _SE, _SE, _I, c_double_p, c_int64_p]),
    'b2ins_diag_noise_plan_ex': (_I, [_D, _L, _L, _SE, _SE, _NT, _NT, _I, c_double_p, c_int64_p]),
    'b2ins_diag_fastmath_f64': (_I, [_I, _L, _P, _P, _P, _P]),
    'b2ins_diag_philox': (_I, [_L, _P, _P]),
    'b2ins_diag_normal_from_words': (_I, [_L, _P, _P]),
}

# function codes of b2ins_diag_fastmath_f64 (include/b2ins.h B2INS_FM_*)
FASTMATH_FNS = ('rcp_nr', 'div_nr', 'sqrt_nr', 'rsqrt_nr', 'sincos_bounded', 'sincos_angle', 'sincospi_2u',
                'log_unit')

_lib = None
_load_error = None       # a failed build is not retried in the same process (every caller gets the same error)


def lib_path():
    return _build.LIB


def load():
    """Load libb2ins.so (building it first if nvcc is here and it is stale)."""
    global _lib, _load_error
    if _lib is not None:
        return _lib
    if _load_error is not None:
        raise B2insError(_load_error)
    path = lib_path()
    if _build.stale():          # missing, or built from other sources than the ones in this tree
        try:
            _build.build()
        except Exception as e:  # no nvcc on this box and no usable prebuilt library
            if not os.path.exists(path):
                _load_error = 'libb2ins.so is missing and could not be built: %s' % e
            else:
                _load_error = 'libb2ins.so was built from other sources and could not be rebuilt: %s' % e
            raise B2insError(_load_error)
    elif _build.LAST_BUILD == 'not checked':
        _build.LAST_BUILD = 'reused'
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the ABI is incomplete
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def mc_shape(lanes, ref_frame=1):
    """'P,WI,split' of the fused Monte-Carlo launch for a lane-group width and a reference frame
    ('0' = single-warp form)."""
    out = (ctypes.c_int * 3)()
    check(load().b2ins_diag_mc_shape(int(lanes), int(ref_frame), out))
    return '%d,%d,%d' % (out[0], out[1], out[2]) if out[0] else '0'


PSD_PLANS = ('direct', 'radix2', 'bluestein')


def psd_plan(n):
    """(plan, P) of K5 for a series of n samples: 'direct' (P = 0), 'radix2' or 'bluestein' (P = the
    transform length)."""
    P = ctypes.c_int(0)
    rc = load().b2ins_diag_psd_plan(int(n), ctypes.byref(P))
    if rc < 0:
        raise ValueError('b2ins: ' + load().b2ins_last_error().decode('utf-8', 'replace'))
    return PSD_PLANS[rc], P.value


def noise_plan(fs, runs, n, gyro_err, accel_err, sm_count=0):
    """K1's (and K9's) digested Gauss-Markov coefficients and time segmentation for `runs` runs of n samples
    on sm_count SMs (0: the current device): {'gm_a', 'gm_b', 'wd': [6] (accel xyz, gyro xyz), 'nseg',
    'seg_len', 'pass1_len'}.  gyro_err / accel_err: imu_model dicts, as engine.imu_noise takes them."""
    ge, ae = sensor_err(gyro_err, 'arw'), sensor_err(accel_err, 'vrw')
    coef = np.zeros(18)
    plan = np.zeros(3, dtype=np.int64)
    check(load().b2ins_diag_noise_plan_ex(float(fs), int(runs), int(n), ctypes.byref(ge), ctypes.byref(ae),
                                           noise_terms(gyro_err), noise_terms(accel_err), int(sm_count),
                                           coef.ctypes.data_as(c_double_p), plan.ctypes.data_as(c_int64_p)))
    return {'gm_a': coef[0:6], 'gm_b': coef[6:12], 'wd': coef[12:18], 'nseg': int(plan[0]),
            'seg_len': int(plan[1]), 'pass1_len': int(plan[2])}


def check(rc):
    if rc != OK:
        msg = load().b2ins_last_error().decode('utf-8', 'replace')
        if rc == ERR_ARG:
            raise ValueError('b2ins: ' + msg)
        raise B2insError('b2ins error %d: %s' % (rc, msg))


def host_ptr(a):
    """void* of a C-contiguous float64 numpy array (or None)."""
    if a is None:
        return None
    assert isinstance(a, np.ndarray) and a.dtype == np.float64 and a.flags['C_CONTIGUOUS']
    return a.ctypes.data_as(ctypes.c_void_p)


def sensor_err(err, white_key):
    """imu_model-style dict {'b','b_drift','b_corr',white_key} -> SensorErr."""
    a = np.array([err['b'], err['b_drift'], err['b_corr'], err[white_key]], dtype=np.float64)   # [4][3] = the struct
    assert a.shape == (4, 3)
    return SensorErr.from_buffer_copy(a)


TERM_KEYS = ('q', 'rrw', 'rr')     # an imu_model dict's IEEE Std 952 terms (Q, K, R), SI units


def set_terms(err):
    """The IEEE Std 952 terms an imu_model dict sets: its keys among TERM_KEYS with a non-zero value."""
    return [k for k in TERM_KEYS if k in err and np.any(np.asarray(err[k], dtype=np.float64) != 0.0)]


def noise_terms(err):
    """imu_model dict -> NoiseTerms (absent keys: zero), or None when it has no non-zero term: the _ex entry
    points then run the kernels without terms."""
    if not set_terms(err):
        return None
    t = NoiseTerms()
    for f, k in zip(('q', 'k', 'r'), TERM_KEYS):
        v = np.broadcast_to(np.asarray(err.get(k, 0.0), dtype=np.float64), (3,))
        for c in range(3):
            getattr(t, f)[c] = float(v[c])
    return t


def vib(vib_def, series_ptr=None, series_len=0):
    """Sim.__parse_env-style dict (or None) -> Vib."""
    v = Vib()
    v.type = VIB_NONE
    if vib_def is None:
        return v
    kind = vib_def['type'].lower()
    if kind == 'random':
        v.type = VIB_RANDOM
    elif kind == 'sinusoidal':
        v.type = VIB_SINUSOIDAL
        v.freq = float(vib_def['freq'])
    elif kind == 'psd':
        v.type = VIB_SERIES
        v.series = series_ptr
        v.series_len = int(series_len)
        return v
    else:
        raise ValueError('unknown vibration type %r' % vib_def['type'])
    v.amp[0], v.amp[1], v.amp[2] = float(vib_def['x']), float(vib_def['y']), float(vib_def['z'])
    return v
