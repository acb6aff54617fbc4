"""Device-level Python API over the C ABI (include/b2ins.h).

PyTorch is plumbing here: it owns device memory (float64 CUDA tensors) and the current
stream; every kernel is in csrc/libb2ins.so.  All functions are asynchronous on the
current torch stream unless they return host data.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import LAYOUT_RUN_MAJOR, LAYOUT_TIME_MAJOR, LAYOUT_CHANNEL_MAJOR  # noqa: F401
from ._lib import POS_FRAME_LLA, POS_FRAME_NED, POS_FRAME_ECEF  # noqa: F401


def _require_cuda():
    if not torch.cuda.is_available():
        raise _lib.B2insError('no CUDA device: the b2ins engine has no CPU fallback')


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    if t is None:
        return None
    assert t.is_cuda and t.dtype == torch.float64 and t.is_contiguous(), 'need contiguous cuda f64'
    return ctypes.c_void_p(t.data_ptr())


def _reuse(cur, shape, dev):
    """cur if it is a buffer of this shape (results handed back through `out=`), else a new f64 one on dev."""
    if cur is not None and tuple(cur.shape) == tuple(shape):
        return cur
    return torch.empty(shape, dtype=torch.float64, device=dev)


def to_device(a, device=None):
    """numpy / tensor -> contiguous float64 CUDA tensor (H2D copy if needed)."""
    if isinstance(a, torch.Tensor):
        return a.to(device=device or 'cuda', dtype=torch.float64).contiguous()
    a = np.ascontiguousarray(a, dtype=np.float64)
    t = torch.from_numpy(a)
    return t.to(device or 'cuda', non_blocking=t.is_pinned())


def ini_sets_from_plugin(ini_pos_vel_att):
    """FreeIntegration's ini_pos_vel_att ((9|10,) or (9|10, S)) -> [S][rows] row-major."""
    a = np.asarray(ini_pos_vel_att, dtype=np.float64)
    if a.ndim == 1:
        a = a.reshape(-1, 1)
    elif a.ndim != 2:
        raise ValueError('Initial states should be a 1D or 2D numpy array, '
                         'but the dimension is %s.' % a.ndim)
    if a.shape[0] not in (9, 10):
        raise ValueError('Initial states need 9 (or 10 with gravity) rows, got %d' % a.shape[0])
    return np.ascontiguousarray(a.T)


def free_integration(ref_frame, fs, gyro, accel, ini, earth_rot=True, layout=LAYOUT_RUN_MAJOR,
                     run_offset=0, lanes_per_run=0):
    """K2.  gyro, accel: CUDA f64 [R,n,3] (RUN_MAJOR) or [n,3,R] (TIME_MAJOR);
    ini: CUDA f64 [S,9|10].  Returns att, pos, vel in the same layout."""
    _require_cuda()
    lib = _lib.load()
    if layout == LAYOUT_RUN_MAJOR:
        R, n, three = gyro.shape
    else:
        n, three, R = gyro.shape
    assert three == 3 and gyro.shape == accel.shape
    att = torch.empty_like(gyro)
    pos = torch.empty_like(gyro)
    vel = torch.empty_like(gyro)
    _lib.check(lib.b2ins_free_integration_f64(
        int(ref_frame), float(fs), R, n, _ptr(gyro), _ptr(accel), layout, _ptr(ini),
        ini.shape[0], ini.shape[1], int(run_offset), int(bool(earth_rot)),
        _ptr(att), _ptr(pos), _ptr(vel), int(lanes_per_run), _stream()))
    return att, pos, vel


def free_integration_odo(ref_frame, fs, gyro, odo, ini, earth_rot=True, layout=LAYOUT_RUN_MAJOR,
                         run_offset=0, lanes_per_run=0):
    """K2, odometer variant.  gyro [R,n,3] / odo [R,n] (RUN_MAJOR) or [n,3,R] / [n,R]."""
    _require_cuda()
    lib = _lib.load()
    if layout == LAYOUT_RUN_MAJOR:
        R, n, _ = gyro.shape
        assert tuple(odo.shape) == (R, n)
    else:
        n, _, R = gyro.shape
        assert tuple(odo.shape) == (n, R)
    att = torch.empty_like(gyro)
    pos = torch.empty_like(gyro)
    vel = torch.empty_like(gyro)
    _lib.check(lib.b2ins_free_integration_odo_f64(
        int(ref_frame), float(fs), R, n, _ptr(gyro), _ptr(odo), layout, _ptr(ini),
        ini.shape[0], ini.shape[1], int(run_offset), int(bool(earth_rot)),
        _ptr(att), _ptr(pos), _ptr(vel), int(lanes_per_run), _stream()))
    return att, pos, vel


def imu_noise(fs, runs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_offset=0,
              vib_gyro=None, vib_accel=None, layout=LAYOUT_RUN_MAJOR, dump_z=False):
    """K1 (b2ins_imu_noise_rx_f64).  ref_gyro/ref_accel: CUDA f64 [n,3]; *_err: imu_model dicts (a non-zero
    'q', 'rrw' or 'rr' adds the IEEE Std 952 terms, a non-zero 'b_std', 'sf' or 'ma' the run-to-run errors; the
    entry point launches the K1 form with what is set).
    Returns gyro, accel ([R,n,3], [n,3,R] or, LAYOUT_CHANNEL_MAJOR, [R,3,n]) and, if dump_z,
    z [R,n,12]."""
    _require_cuda()
    lib = _lib.load()
    n = ref_gyro.shape[0]
    shape = {LAYOUT_RUN_MAJOR: (runs, n, 3), LAYOUT_TIME_MAJOR: (n, 3, runs),
             LAYOUT_CHANNEL_MAJOR: (runs, 3, n)}[layout]
    gyro = torch.empty(shape, dtype=torch.float64, device=ref_gyro.device)
    accel = torch.empty_like(gyro)
    z = torch.empty((runs, n, 12), dtype=torch.float64, device=ref_gyro.device) if dump_z else None
    ge, ae = _lib.sensor_err(gyro_err, 'arw'), _lib.sensor_err(accel_err, 'vrw')
    vg, va = _lib.vib(vib_gyro), _lib.vib(vib_accel)
    _lib.check(lib.b2ins_imu_noise_rx_f64(
        float(fs), runs, n, _ptr(ref_gyro), _ptr(ref_accel), ctypes.byref(ge), ctypes.byref(ae),
        _lib.noise_terms(gyro_err), _lib.noise_terms(accel_err), ctypes.byref(vg), ctypes.byref(va), int(seed),
        int(run_offset), layout, _ptr(gyro), _ptr(accel), _ptr(z), _lib.run_err(gyro_err), _lib.run_err(accel_err),
        _stream()))
    return (gyro, accel, z) if dump_z else (gyro, accel)


def imu_run_errors(runs, gyro_err, accel_err, seed, run_offset=0):
    """The run-to-run errors K1 and K9 draw for runs run_offset .. run_offset + runs - 1 (b2ins_imu_run_err_f64),
    from the imu_model dicts' 'b_std', 'sf', 'ma' (absent: zero).  Returns CUDA f64 [R, 2, 3, 4]: sensor 0 accel,
    1 gyro; row i = (S[i][0], S[i][1], S[i][2], b_run[i]) with S = diag(sf) + ma."""
    _require_cuda()
    lib = _lib.load()
    out = torch.zeros((runs, 2, 12), dtype=torch.float64, device='cuda')
    _lib.check(lib.b2ins_imu_run_err_f64(int(seed) & 0xFFFFFFFFFFFFFFFF, int(runs), int(run_offset),
                                         _lib.run_err(gyro_err), _lib.run_err(accel_err), _ptr(out), _stream()))
    return torch.cat([out[:, :, :9].reshape(runs, 2, 3, 3), out[:, :, 9:].reshape(runs, 2, 3, 1)], dim=3)


def gps_noise(runs, ref_gps, gps_err, gps_type, seed, run_offset=0):
    """K6: pathgen.gps_gen for `runs` runs.  ref_gps: CUDA f64 [m,6]; gps_err {'stdp','stdv'} [3];
    gps_type 0 (LLA, ref_frame 0) or 1 (xyz).  Returns [R,m,6]."""
    _require_cuda()
    lib = _lib.load()
    m = ref_gps.shape[0]
    out = torch.empty((runs, m, 6), dtype=torch.float64, device=ref_gps.device)
    stdp = np.ascontiguousarray(np.broadcast_to(np.asarray(gps_err['stdp'], dtype=np.float64), (3,)))
    stdv = np.ascontiguousarray(np.broadcast_to(np.asarray(gps_err['stdv'], dtype=np.float64), (3,)))
    _lib.check(lib.b2ins_gps_noise_f64(runs, m, _ptr(ref_gps), _lib.host_ptr(stdp), _lib.host_ptr(stdv),
                                       int(gps_type), int(seed), int(run_offset), _ptr(out), _stream()))
    return out


def mag_noise(runs, ref_mag, mag_err, seed, run_offset=0):
    """K8: pathgen.mag_gen for `runs` runs.  ref_mag: CUDA f64 [n,3] (uT, body frame); mag_err
    {'si' [3,3], 'hi' [3], 'std' [3]} (uT).  Returns [R,n,3]."""
    _require_cuda()
    lib = _lib.load()
    n = ref_mag.shape[0]
    out = torch.empty((runs, n, 3), dtype=torch.float64, device=ref_mag.device)
    si = np.ascontiguousarray(np.asarray(mag_err['si'], dtype=np.float64).reshape(3, 3))
    hi = np.ascontiguousarray(np.broadcast_to(np.asarray(mag_err['hi'], dtype=np.float64).reshape(-1), (3,)))
    std = np.ascontiguousarray(np.broadcast_to(np.asarray(mag_err['std'], dtype=np.float64).reshape(-1), (3,)))
    _lib.check(lib.b2ins_mag_noise_f64(runs, n, _ptr(ref_mag), _lib.host_ptr(si), _lib.host_ptr(hi),
                                       _lib.host_ptr(std), int(seed), int(run_offset), _ptr(out), _stream()))
    return out


def _segments(segments):
    """((x0, xf), (y0, yf), (z0, zf)) -> the int64[6] the C ABI takes (it checks the ranges)."""
    seg = np.ascontiguousarray(np.asarray(segments, dtype=np.int64).reshape(6))
    return seg, seg.ctypes.data_as(_lib.c_int64_p)


class MagCalResult:
    """Device-side results of one magnetometer-calibration launch (K10)."""

    def __init__(self):
        self.soft_iron = None    # [R,3,3] S: calibrated = S m - hard_iron[0:3]
        self.hard_iron = None    # [R,4] hard iron [uT], field radius [uT]
        self.err = None          # [R,13] calibration error against the generating model (mag_calibrate_mc)
        self.mag_cal = None      # [R,L,3] the segments after the staged corrections (mag_calibrate, want_cal)


def mag_calibrate(segments, mag, want_cal=False):
    """K10 on supplied samples (b2ins_magcal_fed_f64): the soft- and hard-iron calibration of every run of mag
    (CUDA f64 [R,n,3]) from its rotations about x, y and z, segments ((x0, xf), (y0, yf), (z0, zf)) (half-open
    sample ranges, each >= 3 rows inside [0, n)).  want_cal: also mag_cal [R,L,3], the segments stacked after
    the staged corrections.  Asynchronous on the current stream."""
    _require_cuda()
    lib = _lib.load()
    R, n, three = mag.shape
    if three != 3:
        raise ValueError('mag must be [R, n, 3], got %s' % (tuple(mag.shape),))
    seg, segp = _segments(segments)
    res = MagCalResult()
    res.soft_iron = torch.empty((R, 3, 3), dtype=torch.float64, device=mag.device)
    res.hard_iron = torch.empty((R, 4), dtype=torch.float64, device=mag.device)
    if want_cal:
        L = max(0, int((seg[1] - seg[0]) + (seg[3] - seg[2]) + (seg[5] - seg[4])))
        res.mag_cal = torch.empty((R, L, 3), dtype=torch.float64, device=mag.device)
    _lib.check(lib.b2ins_magcal_fed_f64(R, n, segp, _ptr(mag), 3 * n, 3, _ptr(res.soft_iron), _ptr(res.hard_iron),
                                        _ptr(res.mag_cal), _stream()))
    return res


def mag_calibrate_mc(runs, segments, ref_mag, mag_err, seed, run_offset=0, want_err=True):
    """K8 fused into K10 (b2ins_magcal_f64): the calibration of `runs` runs of the magnetometer mag_noise makes
    (same ref_mag [n,3] CUDA f64, mag_err, seed, run_offset), whose samples are regenerated inside the kernel
    and never written.  want_err: res.err [R,13], the error against mag_err (include/b2ins.h)."""
    _require_cuda()
    lib = _lib.load()
    n = ref_mag.shape[0]
    seg, segp = _segments(segments)
    dev = ref_mag.device
    res = MagCalResult()
    res.soft_iron = torch.empty((runs, 3, 3), dtype=torch.float64, device=dev)
    res.hard_iron = torch.empty((runs, 4), dtype=torch.float64, device=dev)
    res.err = torch.empty((runs, 13), dtype=torch.float64, device=dev) if want_err else None
    si = np.ascontiguousarray(np.asarray(mag_err['si'], dtype=np.float64).reshape(3, 3))
    hi = np.ascontiguousarray(np.broadcast_to(np.asarray(mag_err['hi'], dtype=np.float64).reshape(-1), (3,)))
    std = np.ascontiguousarray(np.broadcast_to(np.asarray(mag_err['std'], dtype=np.float64).reshape(-1), (3,)))
    _lib.check(lib.b2ins_magcal_f64(int(runs), n, segp, _ptr(ref_mag), _lib.host_ptr(si), _lib.host_ptr(hi),
                                    _lib.host_ptr(std), int(seed) & 0xFFFFFFFFFFFFFFFF, int(run_offset),
                                    _ptr(res.soft_iron), _ptr(res.hard_iron), _ptr(res.err), _stream()))
    return res


def imu_err_stats(fs, runs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_offset=0,
                  vib_gyro=None, vib_accel=None, stats_start=-1):
    """K9 (b2ins_imu_err_stats_rx_f64): error statistics of the measurements imu_noise would make, reduced
    inside the generator.
    Returns end_err [R,6] (e = meas - ref at the last sample; accel x y z, gyro x y z) and, if
    stats_start >= 0, proc_stats [R,3,6] (max|e|, mean, std over samples >= stats_start), else None."""
    _require_cuda()
    lib = _lib.load()
    n = ref_gyro.shape[0]
    dev = ref_gyro.device
    end_err = torch.empty((runs, 6), dtype=torch.float64, device=dev)
    proc = torch.empty((runs, 3, 6), dtype=torch.float64, device=dev) if stats_start >= 0 else None
    ge, ae = _lib.sensor_err(gyro_err, 'arw'), _lib.sensor_err(accel_err, 'vrw')
    vg, va = _lib.vib(vib_gyro), _lib.vib(vib_accel)
    _lib.check(lib.b2ins_imu_err_stats_rx_f64(
        float(fs), runs, n, _ptr(ref_gyro), _ptr(ref_accel), ctypes.byref(ge), ctypes.byref(ae),
        _lib.noise_terms(gyro_err), _lib.noise_terms(accel_err), ctypes.byref(vg), ctypes.byref(va), int(seed),
        int(run_offset), int(stats_start), _ptr(end_err), _ptr(proc), _lib.run_err(gyro_err), _lib.run_err(accel_err),
        _stream()))
    return end_err, proc


def proc_stats(x, ref, start):
    """K3p: x CUDA f64 [R,m,C], ref [m,C] -> end_err [R,C] (x - ref at row m-1) and proc_stats
    [R,3,C] (max|e|, mean, std over rows >= start)."""
    _require_cuda()
    lib = _lib.load()
    R, m, C = x.shape
    end_err = torch.empty((R, C), dtype=torch.float64, device=x.device)
    proc = torch.empty((R, 3, C), dtype=torch.float64, device=x.device)
    _lib.check(lib.b2ins_proc_stats_f64(R, m, C, _ptr(x), _ptr(ref), int(start), _ptr(end_err), _ptr(proc),
                                        _stream()))
    return end_err, proc


class McResult:
    """Device-side results of one fused Monte-Carlo launch."""

    def __init__(self):
        self.end_err = None      # [R,9] att(wrapped),pos,vel error at the last sample
        self.end_state = None    # [R,9]
        self.proc_stats = None   # [R,3,9] max|e|, mean, std per run (stats_start >= 0)
        self.att = self.pos = self.vel = None   # [dump_runs,n,3]
        self.gyro = self.accel = None           # [dump_runs,n,3]
        self.odo = None                         # [dump_runs,n] (odometer variant)
        self.quat = None                        # [dump_runs,rows,4] att_quat of the kept samples
        self.lanes_per_run = 0


def make_mc_config(ref_frame, fs, n, runs, seed, gyro_err, accel_err, ini_sets, ini_rows,
                   earth_rot=True, run_offset=0, vib_gyro=None, vib_accel=None,
                   lanes_per_run=0, stats_start=-1, dump_runs=0, ini_offset=None,
                   odo_err=None, ref_odo=None, dump_stride=1, proc_pos_frame=0):
    """odo_err {'scale','stdv'} + ref_odo (CUDA f64 [n]) select the odometer variant.
    proc_pos_frame (ref_frame 0): position columns of proc_stats as LLA differences (0), or as
    NED (1) / ECEF (2) metres, the reference's extra_opt 'ned' / 'ecef'.  It is not a field of
    b2ins_mc_config: mc_free_integration passes it to b2ins_mc_free_integration_ex_f64."""
    cfg = _lib.McConfig()
    cfg.ref_frame = int(ref_frame)
    cfg.earth_rot = int(bool(earth_rot))
    cfg.fs = float(fs)
    cfg.n = int(n)
    cfg.runs = int(runs)
    cfg.run_offset = int(run_offset)
    cfg.ini_offset = int(run_offset if ini_offset is None else ini_offset)
    cfg.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    cfg.gyro_err = _lib.sensor_err(gyro_err, 'arw')
    cfg.accel_err = _lib.sensor_err(accel_err, 'vrw')
    cfg.vib_gyro = _lib.vib(vib_gyro)
    cfg.vib_accel = _lib.vib(vib_accel)
    cfg._keep_vib = (vib_gyro, vib_accel)   # assignment copies the structs: keep the series tensors alive
    cfg.ini_sets = int(ini_sets)
    cfg.ini_rows = int(ini_rows)
    cfg.lanes_per_run = int(lanes_per_run)
    cfg.stats_start = int(stats_start)
    cfg.dump_runs = int(dump_runs)
    cfg.dump_stride = int(dump_stride)
    cfg.proc_pos_frame = int(proc_pos_frame)      # a Python attribute beside the struct's fields
    cfg.algo = 0
    if odo_err is not None:
        assert ref_odo is not None and ref_odo.is_cuda and ref_odo.dtype == torch.float64
        cfg.algo = 1
        cfg.odo_scale = float(odo_err['scale'])
        cfg.odo_stdv = float(odo_err['stdv'])
        cfg.ref_odo = ref_odo.data_ptr()
        cfg._keep = ref_odo            # keep the tensor alive with the config
    return cfg


def mc_free_integration(cfg, ref_gyro, ref_accel, ref_nav, ini, want_state=False,
                        dump_nav=False, dump_imu=False, out=None, dump_quat=False):
    """K12: fused noise generation + free integration + per-run errors.
    ref_gyro, ref_accel [n,3]; ref_nav [n,9] (att,pos,vel); ini [S,rows]: CUDA f64.
    `out` may carry a preallocated McResult to reuse buffers."""
    _require_cuda()
    lib = _lib.load()
    dev = ref_gyro.device
    R, n, D = cfg.runs, cfg.n, cfg.dump_runs
    rows = -(-n // max(1, cfg.dump_stride))          # histories keep every dump_stride-th sample
    res = out or McResult()
    res.end_err = _reuse(res.end_err, (R, 9), dev)
    res.end_state = _reuse(res.end_state, (R, 9), dev) if want_state else None
    res.proc_stats = _reuse(res.proc_stats, (R, 3, 9), dev) if cfg.stats_start >= 0 else None
    if dump_nav and D > 0:
        res.att, res.pos, res.vel = (_reuse(res.att, (D, rows, 3), dev), _reuse(res.pos, (D, rows, 3), dev),
                                     _reuse(res.vel, (D, rows, 3), dev))
        res.quat = _reuse(res.quat, (D, rows, 4), dev) if dump_quat else None
    else:
        res.att = res.pos = res.vel = res.quat = None
    if dump_imu and D > 0:
        res.gyro, res.accel = _reuse(res.gyro, (D, rows, 3), dev), _reuse(res.accel, (D, rows, 3), dev)
        res.odo = _reuse(res.odo, (D, rows), dev) if cfg.algo == 1 else None
    else:
        res.gyro = res.accel = res.odo = None
    cfg.dump_odo = res.odo.data_ptr() if res.odo is not None else None
    cfg.dump_quat = res.quat.data_ptr() if res.quat is not None else None
    _lib.check(lib.b2ins_mc_free_integration_ex_f64(
        ctypes.byref(cfg), getattr(cfg, 'proc_pos_frame', POS_FRAME_LLA),
        _ptr(ref_gyro), _ptr(ref_accel), _ptr(ref_nav), _ptr(ini),
        _ptr(res.end_err), _ptr(res.end_state), _ptr(res.proc_stats),
        _ptr(res.att), _ptr(res.pos), _ptr(res.vel), _ptr(res.gyro), _ptr(res.accel), _stream()))
    return res


class McPlan:
    """b2ins_mc_plan: persistent device + pinned buffers and a stream for one experiment
    shape; run() = stage, H2D, K12, K3, D2H, sync (the low-latency host path of Sim.run)."""

    def __init__(self, n, max_runs, ini_sets, ini_rows):
        _require_cuda()
        self._lib = _lib.load()
        self._h = ctypes.c_void_p()
        self.n, self.max_runs, self.ini_sets, self.ini_rows = int(n), int(max_runs), int(ini_sets), int(ini_rows)
        self.device = torch.cuda.current_device()
        _lib.check(self._lib.b2ins_mc_plan_create(self.n, self.max_runs, self.ini_sets,
                                                  self.ini_rows, ctypes.byref(self._h)))

    def run(self, cfg, ref_gyro, ref_accel, ref_nav_end, ini, want_err=True, want_stats=True):
        """Host float64 C-contiguous arrays in (ref_nav_end: the 9 values att,pos,vel of the true
        trajectory at its last sample); (end_err [runs,9] or None, stats [3,9] or None) out."""
        hp = _lib.host_ptr
        stats = np.empty((3, 9)) if want_stats else None
        err = np.empty((cfg.runs, 9)) if want_err else None
        _lib.check(self._lib.b2ins_mc_plan_run(self._h, ctypes.byref(cfg), hp(ref_gyro), hp(ref_accel),
                                               hp(ref_nav_end), hp(ini), hp(err), hp(stats)))
        return err, stats

    def err_device_ptr(self):
        """Device address of the plan's end_err buffer (multi-GPU statistics exchange)."""
        return self._lib.b2ins_mc_plan_err_device(self._h)

    def stream_ptr(self):
        return self._lib.b2ins_mc_plan_stream(self._h)

    def close(self):
        if self._h:
            self._lib.b2ins_mc_plan_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_plan_cache = {}


def get_plan(n, runs, ini_sets, ini_rows):
    """A cached plan that fits (n, runs, ini layout) on the current device."""
    _require_cuda()
    key = (torch.cuda.current_device(), int(n), int(ini_sets), int(ini_rows))
    plan = _plan_cache.get(key)
    if plan is None or plan.max_runs < runs:
        if plan is not None:
            plan.close()
        plan = McPlan(n, runs, ini_sets, ini_rows)
        _plan_cache[key] = plan
    return plan


def f64c(a):
    """C-contiguous float64 numpy view/copy of a."""
    return np.ascontiguousarray(a, dtype=np.float64)


_ws_cache = {}


def _stats_ws(ncomp, dev):
    key = (ncomp, str(dev))
    if key not in _ws_cache:
        nbytes = _lib.load().b2ins_error_stats_workspace_bytes(ncomp)
        _ws_cache[key] = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device=dev)
    return _ws_cache[key]


def error_stats(err):
    """K3 on one shard.  err: CUDA f64 [R, ncomp] -> stats [3, ncomp] = max|e|, mean, std."""
    _require_cuda()
    lib = _lib.load()
    R, nc = err.shape
    stats = torch.empty((3, nc), dtype=torch.float64, device=err.device)
    _lib.check(lib.b2ins_error_stats_f64(R, nc, _ptr(err), _ptr(stats),
                                         _ptr(_stats_ws(nc, err.device)), _stream()))
    return stats


def psd_series(fs, n, runs, sensor, vib_def, seed, run_offset=0):
    """K5.  vib_def: {'type': 'psd', 'freq': (L0,), 'x','y','z': (L0,)} (Sim.__parse_env output).
    Returns the device series [runs, 3, N] and N (hand both to a Vib of type VIB_SERIES)."""
    _require_cuda()
    lib = _lib.load()
    freq = to_device(vib_def['freq'])
    if fs < 2.0 * float(vib_def['freq'][-1]) or fs < 0.0:
        raise ValueError('PSD table exceeds fs/2 (time_series_from_psd.py:33-34)')
    sxx = to_device(np.stack([vib_def['x'], vib_def['y'], vib_def['z']]))
    N = lib.b2ins_psd_series_len(int(n))
    out = []
    for r0 in range(0, runs, 16384):                       # grid.y limit per launch
        r1 = min(runs, r0 + 16384)
        series = torch.empty((r1 - r0, 3, N), dtype=torch.float64, device=freq.device)
        ws = torch.empty(lib.b2ins_psd_workspace_bytes(int(n), r1 - r0) // 8 + 1, dtype=torch.float64,
                         device=freq.device)
        _lib.check(lib.b2ins_psd_series_f64(float(fs), int(n), r1 - r0, int(sensor), freq.numel(),
                                            _ptr(freq), _ptr(sxx), int(seed), int(run_offset) + r0,
                                            _ptr(series), _ptr(ws), _stream()))
        out.append(series)
    return (out[0] if len(out) == 1 else torch.cat(out)), N


def vib_series(series, N):
    """A Vib of type VIB_SERIES over a device series [runs, 3, N]."""
    v = _lib.Vib()
    v.type = _lib.VIB_SERIES
    v.series = series.data_ptr()
    v.series_len = int(N)
    v._keep = series               # the device series lives as long as the Vib does
    return v


def allan_num_tau(n, fs):
    lib = _lib.load()
    m = (ctypes.c_int64 * 128)()
    k = lib.b2ins_allan_num_tau(int(n), float(fs), m, 128)
    return list(m[:k])


def allan_taus(n, fs):
    """tau [s] of the cluster sizes allan_var uses for n samples at fs (allan.py:37-43, :58)."""
    return np.asarray(allan_num_tau(n, fs), dtype=np.float64) / float(fs)


def _outer_stride(n, inner, outer_stride, sample_stride):
    """outer_stride of the series addressing when the caller gives none: series after series (inner == 1), or
    groups of `inner` interleaved series after one another."""
    if outer_stride is not None:
        return outer_stride
    return n * sample_stride if inner == 1 else n * inner


def _variance(symbol, workspace_symbol, fs, x, n, nseries, inner, outer_stride, sample_stride):
    """K4 or K4o's two forms through the C ABI entry `symbol`: var [nseries, ntau], tau [ntau] (CUDA)."""
    _require_cuda()
    lib = _lib.load()
    outer_stride = _outer_stride(n, inner, outer_stride, sample_stride)
    ntau = len(allan_num_tau(n, fs))
    var = torch.zeros((nseries, ntau), dtype=torch.float64, device=x.device)
    tau = torch.zeros((ntau,), dtype=torch.float64, device=x.device)
    if ntau == 0 or nseries == 0:
        return var, tau
    ws = torch.empty(getattr(lib, workspace_symbol)(int(n), int(nseries)) // 8 + 1, dtype=torch.float64,
                     device=x.device)
    _lib.check(getattr(lib, symbol)(float(fs), int(n), int(nseries), _ptr(x), int(inner), int(outer_stride),
                                    int(sample_stride), _ptr(var), _ptr(tau), _ptr(ws), _stream()))
    return var, tau


def allan(fs, x, n, nseries, inner=1, outer_stride=None, sample_stride=1):
    """K4.  x: CUDA f64 buffer holding `nseries` series of n samples; series s, sample t at
    x.flat[(s // inner) * outer_stride + (s % inner) + t * sample_stride].
    Returns avar [nseries, ntau], tau [ntau] (CUDA)."""
    return _variance('b2ins_allan_f64', 'b2ins_allan_workspace_bytes', fs, x, n, nseries, inner, outer_stride,
                     sample_stride)


def oallan_workspace_bytes(n, nseries):
    """Device scratch of engine.oallan for `nseries` series of n samples (about 16 B per series-sample)."""
    return int(_lib.load().b2ins_oallan_workspace_bytes(int(n), int(nseries)))


def oallan(fs, x, n, nseries, inner=1, outer_stride=None, sample_stride=1):
    """K4o: overlapping Allan variance on K4's tau grid, same addressing and outputs as allan():
    avar_o(m) = 1/(2 m^2 M) sum_{k<M} (S(k+m, m) - S(k, m))^2, M = n - 2m + 1.
    Returns avar [nseries, ntau], tau [ntau] (CUDA)."""
    return _variance('b2ins_oallan_f64', 'b2ins_oallan_workspace_bytes', fs, x, n, nseries, inner, outer_stride,
                     sample_stride)


def ohadamard(fs, x, n, nseries, inner=1, outer_stride=None, sample_stride=1):
    """K4o's Hadamard form: overlapping Hadamard variance on K4's tau grid, same addressing and outputs
    as allan(): hvar(m) = 1/(6 m^2 H) sum_{k<H} (S(k+2m, m) - 2 S(k+m, m) + S(k, m))^2, H = n - 3m + 1.
    A linear drift of the samples cancels; white noise gives sigma^2 / m, as avar_o does.
    Returns hvar [nseries, ntau], tau [ntau] (CUDA)."""
    return _variance('b2ins_ohadamard_f64', 'b2ins_oallan_workspace_bytes', fs, x, n, nseries, inner, outer_stride,
                     sample_stride)


def allan_fit(fs, n, var, series_stride=None, bin_stride=1, nseries=None):
    """K13: the IEEE Std 952 noise coefficients of Allan variance curves on the grid of n samples at fs, as
    allan / oallan / allan_mc return them (the variance, read in place).  var: CUDA f64, curve s, bin k at
    var.flat[s * series_stride + k * bin_stride] (series_stride None: ntau, so [nseries, ntau] and [runs, 6, ntau]
    are read as they are); nseries None: var.numel() // ntau (with ntau = 0: the product of var's leading
    dimensions).  Returns [nseries, 6] (CUDA): Q, N, B, K, R and B_min (include/b2ins.h, DESIGN.md section 3.13).
    Asynchronous on the current stream."""
    _require_cuda()
    ntau = len(allan_num_tau(n, fs))
    if nseries is None:
        nseries = var.numel() // ntau if ntau else int(np.prod(var.shape[:-1]))
    nseries = int(nseries)
    series_stride = ntau if series_stride is None else int(series_stride)
    if nseries and ntau and (nseries - 1) * series_stride + (ntau - 1) * int(bin_stride) >= var.numel():
        raise ValueError('%d curves of %d bins with strides (%d, %d) do not fit in %d values'
                         % (nseries, ntau, series_stride, bin_stride, var.numel()))
    out = torch.empty((nseries, 6), dtype=torch.float64, device=var.device)
    _lib.check(_lib.load().b2ins_allan_fit_f64(float(fs), int(n), nseries, _ptr(var) if ntau else None,
                                               int(series_stride), int(bin_stride), _ptr(out), _stream()))
    return out


def welch_workspace_bytes(n, nseries, nperseg, noverlap):
    """Device scratch of engine.welch; negative if nperseg is not a length K11 transforms (or noverlap and n
    give no segment)."""
    return int(_lib.load().b2ins_welch_workspace_bytes(int(n), int(nseries), int(nperseg), int(noverlap)))


def welch(fs, x, n, nseries, nperseg, noverlap, window, inner=1, outer_stride=None, sample_stride=1):
    """K11: scipy.signal.welch(x, fs, window, nperseg, noverlap) (detrend='constant', scaling='density',
    one-sided, nfft = nperseg) of `nseries` series of n samples, addressed as in allan().  window: [nperseg]
    floats.  Returns psd [nseries, nperseg // 2 + 1], freq [nperseg // 2 + 1] (CUDA)."""
    _require_cuda()
    outer_stride = _outer_stride(n, inner, outer_stride, sample_stride)
    L = int(nperseg) // 2 + 1
    w = to_device(window, x.device)
    if w.shape != (int(nperseg),):
        raise ValueError('window must have shape (%d,), got %s' % (int(nperseg), tuple(w.shape)))
    psd = torch.empty((nseries, L), dtype=torch.float64, device=x.device)
    freq = torch.empty((L,), dtype=torch.float64, device=x.device)
    ws = torch.empty(max(welch_workspace_bytes(n, nseries, nperseg, noverlap), 8) // 8 + 1, dtype=torch.float64,
                     device=x.device)
    _lib.check(_lib.load().b2ins_welch_f64(float(fs), int(n), int(nseries), _ptr(x), int(inner), int(outer_stride),
                                           int(sample_stride), int(nperseg), int(noverlap), _ptr(w), _ptr(psd),
                                           _ptr(freq), _ptr(ws), _stream()))
    return psd, freq


def allan_mc(fs, runs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_offset=0):
    """K1 fused into K4: Allan variance of `runs` Monte-Carlo runs x 6 channels whose series are
    generated inside the tau-binning kernel (never written).  ref_gyro, ref_accel: CUDA f64 [n,3].
    Returns avar [runs, 6, ntau] (channels: accel x y z, gyro x y z) and tau [ntau] (CUDA)."""
    _require_cuda()
    lib = _lib.load()
    n = ref_gyro.shape[0]
    ntau = len(allan_num_tau(n, fs))
    avar = torch.zeros((runs, 6, ntau), dtype=torch.float64, device=ref_gyro.device)
    tau = torch.zeros((ntau,), dtype=torch.float64, device=ref_gyro.device)
    if ntau == 0 or runs == 0:
        return avar, tau
    ws = torch.empty(lib.b2ins_allan_workspace_bytes(n, runs * 6) // 8 + 1, dtype=torch.float64,
                     device=ref_gyro.device)
    ge, ae = _lib.sensor_err(gyro_err, 'arw'), _lib.sensor_err(accel_err, 'vrw')
    _lib.check(lib.b2ins_allan_mc_f64(float(fs), int(n), int(runs), _ptr(ref_gyro), _ptr(ref_accel),
                                      ctypes.byref(ge), ctypes.byref(ae), int(seed), int(run_offset),
                                      _ptr(avar), _ptr(tau), _ptr(ws), _stream()))
    return avar, tau


def _ekf_config(fs, n, runs, m, seed, gyro_err, accel_err, gps_err, ini, run_offset, ini_att_std, earth_rot,
                stats_start, dump_runs, dump_stride, vel_rw, att_rw):
    """b2ins_ekf_config of one K7 launch."""
    cfg = _lib.EkfConfig()
    cfg.fs, cfg.n, cfg.runs, cfg.run_offset, cfg.m = float(fs), int(n), int(runs), int(run_offset), int(m)
    cfg.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    cfg.gyro_err = _lib.sensor_err(gyro_err, 'arw')
    cfg.accel_err = _lib.sensor_err(accel_err, 'vrw')
    stdp = np.broadcast_to(np.asarray(gps_err['stdp'], dtype=np.float64), (3,))
    stdv = np.broadcast_to(np.asarray(gps_err['stdv'], dtype=np.float64), (3,))
    ini = np.asarray(ini, dtype=np.float64).reshape(-1)
    for c in range(3):
        cfg.gps_stdp[c], cfg.gps_stdv[c] = float(stdp[c]), float(stdv[c])
        cfg.ini_att_std[c] = float(ini_att_std[c])
    for c in range(9):
        cfg.ini[c] = float(ini[c])
    cfg.stats_start, cfg.dump_runs, cfg.dump_stride = int(stats_start), int(dump_runs), int(dump_stride)
    cfg.earth_rot = int(bool(earth_rot))
    cfg.vel_rw, cfg.att_rw = float(vel_rw), float(att_rw)
    return cfg


def _ekf_result(out, runs, n, dump_runs, dump_stride, dev, end_err):
    """The EkfResult buffers of one K7 launch (those of `out` where they fit); consist is the caller's."""
    res = out or EkfResult()
    res.end_err = _reuse(res.end_err, (runs, 9), dev) if end_err else None
    res.end_bias = _reuse(res.end_bias, (runs, 6), dev)
    if dump_runs > 0:
        rows = -(-n // max(1, int(dump_stride)))
        res.att, res.pos, res.vel, res.wb, res.ab = (_reuse(getattr(res, k), (dump_runs, rows, 3), dev)
                                                     for k in ('att', 'pos', 'vel', 'wb', 'ab'))
    else:
        res.att = res.pos = res.vel = res.wb = res.ab = None
    return res


ALIGN_N = 10       # alignment: accelerometer samples averaged for roll and pitch (ins_loose.py:72)


def align_fix(gps_idx, gps_vis):
    """(fix row, start sample) of an aligned filter (b2ins_ekf_align): the latest visible GPS row at or before
    sample ALIGN_N - 1, else the first visible row after it, and max(ALIGN_N - 1, its sample); (None, None)
    without a visible row.  gps_idx, gps_vis: host arrays [m]."""
    gps_idx = np.asarray(gps_idx, dtype=np.int64).reshape(-1)
    vis = np.nonzero(np.asarray(gps_vis, dtype=np.float64).reshape(-1) > 0.0)[0]
    if vis.size == 0:
        return None, None
    before = vis[gps_idx[vis] <= ALIGN_N - 1]
    j = int(before[-1]) if before.size else int(vis[0])
    return j, max(ALIGN_N - 1, int(gps_idx[j]))


def _ekf_ini(ini, align):
    """The initial state of a K7 launch: ini, which an aligned launch does not use (zeros if None)."""
    if ini is None:
        if align is None:
            raise ValueError('the filter needs its initial state ini (or align)')
        return np.zeros(9)
    return ini


def _ekf_align(align):
    """b2ins_ekf_align of align = (yaw, yaw_var): yaw a heading [rad] or 'gps' (the fix row's course)."""
    a = _lib.EkfAlign()
    yaw, yaw_var = align
    if isinstance(yaw, str):
        if yaw != 'gps':
            raise ValueError("align yaw must be a heading in rad or 'gps'")
        a.mode = _lib.ALIGN_GPS
    else:
        a.mode, a.yaw, a.yaw_var = _lib.ALIGN_YAW, float(yaw), float(yaw_var)
    return a


class EkfResult:
    """Device-side results of one loosely-coupled-filter launch (K7)."""

    def __init__(self):
        self.end_err = None      # [R,9] att (wrapped), pos (LLA), vel error at the last sample
        self.end_bias = None     # [R,6] gyro, accel bias estimates at the last sample
        self.consist = None      # [R,19] NEES sums (pos, vel, att), inside-3-sigma counts [15], epochs
        self.proc_stats = None   # [R,3,9] max|e|, mean, std of att, pos, vel per run (proc_start given)
        self.end_bias_err = None # [R,6] gyro, accel bias estimates minus the true biases at the last sample (bias_err)
        self.att = self.pos = self.vel = self.wb = self.ab = None   # [dump_runs,rows,3]
        self.start = 0           # first sample of the filter (aligned: the fix sample, align_fix)


def ins_loose(fs, runs, seed, gyro_err, accel_err, gps_err, ini, ref_gyro, ref_accel, ref_nav, ref_gps,
              gps_idx, gps_vis, run_offset=0, ini_att_std=(0.02, 0.005, 0.005), earth_rot=True,
              stats_start=0, dump_runs=0, dump_stride=1, out=None, vel_rw=0.02, att_rw=0.0,
              vib_gyro=None, vib_accel=None, proc_start=None, proc_pos_frame=0, align=None, bias_err=False):
    """K7: Monte-Carlo loosely-coupled GNSS/INS filter (the spec: DESIGN.md section 11; csrc/ekf_kernel.cuh).
    ref_gyro, ref_accel [n,3], ref_nav [n,9], ref_gps [m,6], gps_vis [m]: CUDA f64; gps_idx [m]: CUDA
    int64 (IMU sample index of every GPS row).  ini: the 9 true initial values (LLA, body velocity, Euler
    angles).  vib_gyro / vib_accel: the vibration of the measurements the filter sees, as imu_noise takes
    them (a parsed dict, or a Vib such as vib_series over K5 series of exactly these runs); the filter
    model does not include it (vel_rw / att_rw, DESIGN.md section 11).  proc_start (sample index in [0, n)):
    also res.proc_stats [R,3,9], the per-run process-error statistics of samples >= proc_start, positions as
    POS_FRAME_* proc_pos_frame (b2ins_ins_loose_proc_f64); every other output is unchanged.  align = (yaw, yaw_var):
    every run initialises itself from its measurements (b2ins_ins_loose_align_f64; yaw a heading [rad] with
    variance yaw_var, or 'gps'); ini is then unused, res.start is the fix sample (align_fix), the consistency
    record takes the epochs after it and proc statistics start at max(proc_start, res.start).  The IMU's turn-on bias
    'b_std' (imu_model; 'sf' and 'ma' are refused) is drawn per run as K1 draws it and is in the filter's P0 and in
    the consistency record's truth (b2ins_ins_loose_rx_f64).  bias_err: also res.end_bias_err [R,6], the bias
    estimates minus the true biases at the last sample.  Asynchronous on the current stream (with align, after one
    host copy of gps_idx / gps_vis)."""
    _require_cuda()
    lib = _lib.load()
    n, m = ref_gyro.shape[0], ref_gps.shape[0]
    dev = ref_gyro.device
    assert gps_idx.dtype == torch.int64 and gps_idx.is_cuda and gps_idx.is_contiguous()
    cfg = _ekf_config(fs, n, runs, m, seed, gyro_err, accel_err, gps_err, _ekf_ini(ini, align), run_offset,
                      ini_att_std, earth_rot, stats_start, dump_runs, dump_stride, vel_rw, att_rw)
    # Vib structs are passed by pointer; a VIB_SERIES Vib keeps its series tensor alive through the call
    vg, va = _lib.vib(vib_gyro), _lib.vib(vib_accel)
    res = _ekf_result(out, runs, n, dump_runs, dump_stride, dev, end_err=True)
    res.consist = _reuse(res.consist, (runs, 19), dev)
    res.proc_stats = None if proc_start is None else _reuse(res.proc_stats, (runs, 3, 9), dev)
    res.end_bias_err = _reuse(res.end_bias_err, (runs, 6), dev) if bias_err else None
    refs = (_ptr(ref_gyro), _ptr(ref_accel), _ptr(ref_nav), _ptr(ref_gps), ctypes.c_void_p(gps_idx.data_ptr()),
            _ptr(gps_vis), _ptr(res.end_err), _ptr(res.end_bias), _ptr(res.consist))
    dumps = (_ptr(res.att), _ptr(res.pos), _ptr(res.vel), _ptr(res.wb), _ptr(res.ab))
    if align is not None:
        res.start = align_fix(gps_idx.cpu().numpy(), gps_vis.cpu().numpy())[1]
    ps = -1 if proc_start is None else int(proc_start)
    gr, ar = _lib.run_err(gyro_err), _lib.run_err(accel_err)
    if gr is not None or ar is not None or bias_err:
        _lib.check(lib.b2ins_ins_loose_rx_f64(
            ctypes.byref(cfg), None if align is None else ctypes.byref(_ekf_align(align)), ctypes.byref(vg),
            ctypes.byref(va), ps, int(proc_pos_frame), *refs, _ptr(res.proc_stats), *dumps, gr, ar,
            _ptr(res.end_bias_err), _stream()))
    elif align is not None:
        _lib.check(lib.b2ins_ins_loose_align_f64(
            ctypes.byref(cfg), ctypes.byref(_ekf_align(align)), ctypes.byref(vg), ctypes.byref(va), ps,
            int(proc_pos_frame), *refs, _ptr(res.proc_stats), *dumps, _stream()))
    elif proc_start is None:
        _lib.check(lib.b2ins_ins_loose_ex_f64(ctypes.byref(cfg), ctypes.byref(vg), ctypes.byref(va), *refs, *dumps,
                                              _stream()))
    else:
        _lib.check(lib.b2ins_ins_loose_proc_f64(ctypes.byref(cfg), ctypes.byref(vg), ctypes.byref(va), ps,
                                                int(proc_pos_frame), *refs, _ptr(res.proc_stats), *dumps, _stream()))
    return res


def ins_loose_fed(fs, gyro, accel, gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err, ini, seed=0, ini_draw=False,
                  run_offset=0, ini_att_std=(0.02, 0.005, 0.005), earth_rot=True, ref_nav=None, dump_runs=0,
                  dump_stride=1, out=None, vel_rw=0.02, att_rw=0.0, align=None):
    """K7 on supplied measurements (b2ins_ins_loose_fed_f64): gyro, accel [R,n,3] and gps [R,m,6] (LLA rad, m;
    NED m/s) CUDA f64, run-major; gps_idx [m] CUDA int64, strictly ascending IMU sample indices of the GPS rows;
    gps_vis [m] CUDA f64.  gyro_err / accel_err / gps_err are the filter's model (Q, R, P0) only.  Every run
    starts at ini, plus with ini_draw the P0 draw of global run run_offset + r under seed (the generated
    experiment's draw).  ref_nav [n,9] (optional): end_err as engine.ins_loose makes it.  Returns an
    EkfResult without consist (and without end_err when ref_nav is None).  align = (yaw, yaw_var): every run
    initialises itself from its measurements instead (b2ins_ins_loose_fed_align_f64; ini, seed and ini_draw are
    unused), res.start is the fix sample.  The model's turn-on bias 'b_std' enters P0 as in ins_loose (the
    measurements carry each run's bias); its 'sf' and 'ma' are not filter states and are not used.  Asynchronous on
    the current stream."""
    _require_cuda()
    lib = _lib.load()
    R, n, three = gyro.shape
    m = gps.shape[1]
    if three != 3 or tuple(accel.shape) != (R, n, 3) or tuple(gps.shape) != (R, m, 6):
        raise ValueError('gyro, accel must be [R, n, 3] and gps [R, m, 6]; got %s, %s, %s'
                         % (tuple(gyro.shape), tuple(accel.shape), tuple(gps.shape)))
    if tuple(gps_idx.shape) != (m,) or tuple(gps_vis.shape) != (m,):
        raise ValueError('gps_idx and gps_vis need one entry per GPS row (%d)' % m)
    if ref_nav is not None and tuple(ref_nav.shape) != (n, 9):
        raise ValueError('ref_nav must be [n, 9]')
    assert gps_idx.dtype == torch.int64 and gps_idx.is_cuda and gps_idx.is_contiguous()
    cfg = _ekf_config(fs, n, R, m, seed, gyro_err, accel_err, gps_err, _ekf_ini(ini, align), run_offset, ini_att_std,
                      earth_rot, -1, dump_runs, dump_stride, vel_rw, att_rw)
    res = _ekf_result(out, R, n, dump_runs, dump_stride, gyro.device, end_err=ref_nav is not None)
    res.consist = None
    if align is not None:
        res.start = align_fix(gps_idx.cpu().numpy(), gps_vis.cpu().numpy())[1]
    _lib.check(lib.b2ins_ins_loose_fed_rx_f64(
        ctypes.byref(cfg), None if align is None else ctypes.byref(_ekf_align(align)),
        int(bool(ini_draw)) if align is None else 0, _ptr(gyro), _ptr(accel), _ptr(gps),
        ctypes.c_void_p(gps_idx.data_ptr()), _ptr(gps_vis), _ptr(ref_nav), _ptr(res.end_err), _ptr(res.end_bias),
        _ptr(res.att), _ptr(res.pos), _ptr(res.vel), _ptr(res.wb), _ptr(res.ab), _turn_on_bias(gyro_err),
        _turn_on_bias(accel_err), _stream()))
    return res


def _turn_on_bias(err):
    """RunErr of an imu_model dict's turn-on bias 'b_std' alone (None without one): what the fed filter's model
    takes of the run-to-run errors."""
    return _lib.run_err({'b_std': err['b_std']} if 'b_std' in err else {})
