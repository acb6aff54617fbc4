"""Sim -- Monte-Carlo simulation facade with the interface of gnss_ins_sim.sim.ins_sim.Sim
(ins_sim.py:27-337: same constructor arguments, run(num_times), results(...),
get_data(names), the same data names / run keys / units), whose Monte-Carlo loops
(loop A ins_sim.py:490-506, loop B ins_algo_manager.py:73-95) run as CUDA kernels.

What stays on the CPU, by design (BASELINE north_star: "pathgen.path_gen stays CPU-side
and its reference trajectory is broadcast once"): the true trajectory.  `motion_def` is
  * a trajectory: dict / .npz path with time, ref_pos, ref_vel, ref_att, ref_accel,
    ref_gyro (what pathgen.path_gen returns, e.g. tests/golden/traj_*.npz), or
  * a motion-definition .csv / string exactly as the reference takes it; it is turned into a
    trajectory on the host by gnss_ins_sim_b200.pathgen.path_gen (C++ restatement of the
    reference's path generator, identical output, ~200x faster).

Dispatch on `algorithm`:
  * gnss_ins_sim_b200 FreeIntegration  -> K12, the fused noise+integration+error kernel;
    only per-run end-point errors, their ensemble statistics (and, on request, per-run
    process-error statistics) leave the device.  Per-run histories are materialised
    lazily: counter-based Philox makes any run reproducible in isolation, so
    get_data(['pos'])[0]['algo0_7'] re-runs just run 7 with history output on.
  * gnss_ins_sim_b200 Allan            -> K1 (noise) + K4 (Allan variance) per run block; fit=True adds
                                         K13 (noise identification) on the device curves.
  * gnss_ins_sim_b200 Psd              -> K1 (noise) + K11 (Welch power spectral density) per run block.
  * gnss_ins_sim_b200 MagCal           -> K8's samples regenerated inside K10 (magnetometer calibration).
  * any other reference-style plugin   -> K1 generates gyro/accel (K8 the magnetometer of a
    9-axis IMU) on the device, the plugin's own .run() is called per run on the host
    (compatibility path).
  * None                               -> sensor data only.
Multi-GPU: runs are sharded by rank when torch.distributed is initialised (dist.py).
"""
import copy
import math
import os
import weakref
from collections.abc import Mapping

import numpy as np
import torch

from . import _lib, engine, dist, logged
from .free_integration import FreeIntegration
from .free_integration_odo import FreeIntegration as FreeIntegrationOdo
from .series_analysis import SeriesEstimator
from .ins_loose import InsLoose, gps_sample_index
from .mag_calibrate import MagCal, check_segments

D2R = math.pi / 180
R2D = 180 / math.pi
_RE = 6378137.0
_E_SQR = 0.0818191908426215 ** 2


# ------------------------------------------------------------------ helpers ---
def parse_env(env, fs):
    """Vibration DSL -> dict, as Sim.__parse_env (ins_sim.py:642-701):
    '[x y z](g|d)-random', '[x y z](g|d)-<f>Hz-sinusoidal', or (n,4) PSD array."""
    if env is None:
        return None
    if isinstance(env, np.ndarray):
        if env.ndim == 2 and env.shape[1] == 4:
            m = env.shape[0]
            if env[-1, 0] > 0.5 * fs:
                m = np.where(env[:, 0] > 0.5 * fs)[0][0]
            return {'type': 'psd', 'freq': env[:m, 0], 'x': env[:m, 1], 'y': env[:m, 2],
                    'z': env[:m, 3]}
        raise TypeError('env should be of size (n,2)')
    if not isinstance(env, str):
        raise TypeError('env should be a string or a numpy array of size (n,2)')
    text = env.lower()
    out = {}
    if 'random' in text:
        out['type'] = 'random'
        text = text.replace('-random', '')
    elif 'sinusoidal' in text:
        out['type'] = 'sinusoidal'
        text = text.replace('-sinusoidal', '')
        if text[-2:] != 'hz':
            raise ValueError('env = \'%s\' is not valid (No vib freq).' % env)
        cut = text.find('-')
        try:
            out['freq'] = math.fabs(float(text[cut + 1:-2]))
        except ValueError:
            raise ValueError('env = \'%s\' is not valid (invalid vib freq).' % env)
        text = text[:cut]
    else:
        raise ValueError('env = \'%s\' is not valid.' % env)
    scale = 1.0
    if text[-1] == 'g':
        scale, text = 9.8, text[:-1]
    elif text[-1] == 'd':
        scale, text = D2R, text[:-1]
    try:
        amp = scale * np.array(text[1:-1].split(' '), dtype='float64')
        out['x'], out['y'], out['z'] = amp[0], amp[1], amp[2]
    except (ValueError, IndexError):
        raise ValueError('Cannot convert \'%s\' to float' % env)
    return out


def lla2ecef(lla):
    """geoparams.lla2ecef_batch (geoparams.py:89-113), host side, for 'ned' error option."""
    lla = np.atleast_2d(np.asarray(lla, dtype=np.float64))
    sl, cl = np.sin(lla[:, 0]), np.cos(lla[:, 0])
    r = _RE / np.sqrt(1.0 - _E_SQR * sl * sl)
    rho = (r + lla[:, 2]) * cl
    return np.stack([rho * np.cos(lla[:, 1]), rho * np.sin(lla[:, 1]),
                     (r * (1.0 - _E_SQR) + lla[:, 2]) * sl], axis=1)


def ecef_to_ned(lat, lon):
    """attitude.ecef_to_ned (attitude.py: c_ne), rotation ECEF -> local NED."""
    sl, cl, so, co = math.sin(lat), math.cos(lat), math.sin(lon), math.cos(lon)
    return np.array([[-sl * co, -sl * so, cl], [-so, co, 0.0], [-cl * co, -cl * so, -sl]])


def lla_error_metres(x, r, frame):
    """array_error of LLA positions (ins_data_manager.py:543-552), vectorised over samples: x, r [n,3]
    -> lla2ecef(x) - lla2ecef(r) [n,3] (frame 2, ECEF), rotated by ecef_to_ned of every row of r
    (frame 1, NED)."""
    d = lla2ecef(x) - lla2ecef(r)
    if frame == 1:   # the rows of ecef_to_ned(r[i, 0], r[i, 1]) . d[i]
        sl, cl, so, co = np.sin(r[:, 0]), np.cos(r[:, 0]), np.sin(r[:, 1]), np.cos(r[:, 1])
        d = np.stack([-sl * co * d[:, 0] - sl * so * d[:, 1] + cl * d[:, 2],
                      -so * d[:, 0] + co * d[:, 1],
                      -cl * co * d[:, 0] - cl * so * d[:, 1] - sl * d[:, 2]], axis=1)
    return d


def euler2dcm_zyx(att):
    """(3,) yaw, pitch, roll -> the n -> b DCM (attitude.euler2dcm 'zyx' layout)."""
    sy, cy = math.sin(att[0]), math.cos(att[0])
    sp, cp = math.sin(att[1]), math.cos(att[1])
    sr, cr = math.sin(att[2]), math.cos(att[2])
    return np.array([[cp * cy, cp * sy, -sp],
                     [sr * sp * cy - cr * sy, sr * sp * sy + cr * cy, sr * cp],
                     [cr * sp * cy + sr * sy, cr * sp * sy - sr * cy, cr * cp]])


def euler2quat_zyx(att):
    """attitude.euler2quat 'zyx' (attitude.py:188-205), vectorised over rows: (n,3) -> (n,4)
    scalar-first.  The reference associates att_quat with every att_euler it holds
    (ins_sim.py:729-794, a per-sample Python loop that is 22 % of its run time)."""
    att = np.asarray(att, dtype=np.float64)
    c, s = np.cos(0.5 * att), np.sin(0.5 * att)
    return np.stack([c[:, 0] * c[:, 1] * c[:, 2] + s[:, 0] * s[:, 1] * s[:, 2],
                     c[:, 0] * c[:, 1] * s[:, 2] - s[:, 0] * s[:, 1] * c[:, 2],
                     c[:, 0] * s[:, 1] * c[:, 2] + s[:, 0] * c[:, 1] * s[:, 2],
                     s[:, 0] * c[:, 1] * c[:, 2] - c[:, 0] * s[:, 1] * s[:, 2]], axis=1)


class DerivedRuns(Mapping):
    """A per-run view computed from another per-run mapping on access (att_quat from att_euler)."""

    def __init__(self, src, fn):
        self._src, self._fn = src, fn

    def __iter__(self):
        return iter(self._src)

    def __len__(self):
        return len(self._src)

    def __contains__(self, key):
        return key in self._src

    def __getitem__(self, key):
        return self._fn(self._src[key])


def load_trajectory(src):
    """dict / npz path -> dict of float64 arrays with the pathgen names."""
    if isinstance(src, str):
        src = dict(np.load(src, allow_pickle=False))
    need = ('ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')
    alias = {'ref_att': 'ref_att_euler'}
    out = {}
    for k in need:
        key = k if k in src else alias.get(k, k)
        if key not in src:
            raise ValueError('trajectory is missing %r' % k)
        out[k] = np.ascontiguousarray(src[key], dtype=np.float64)
    n = out['ref_gyro'].shape[0]
    for k in need:
        if out[k].shape != (n, 3):
            raise ValueError('trajectory %s must be (n,3)' % k)
    if 'ref_odo' in src:
        out['ref_odo'] = np.ascontiguousarray(src['ref_odo'], dtype=np.float64).reshape(-1)
    if 'ref_mag' in src:
        out['ref_mag'] = np.ascontiguousarray(src['ref_mag'], dtype=np.float64)
        if out['ref_mag'].shape != (n, 3):
            raise ValueError('trajectory ref_mag must be (n,3)')
    if 'time' in src:
        out['time'] = np.asarray(src['time'], dtype=np.float64)
    if 'ini' in src:
        out['ini'] = np.asarray(src['ini'], dtype=np.float64)
    for k in ('gps_time', 'ref_gps', 'gps_visibility'):     # pathgen 'gps' rows, if the caller has them
        if k in src:
            out[k] = np.ascontiguousarray(src[k], dtype=np.float64)
    return out


def trajectory_from_motion_def(fs, motion_def, ref_frame, mode=None, magnetometer=False, odo=False,
                               gps=False, fs_gps=0.0, wmm_file=None, wmm_date=None):
    """Motion-definition csv/string -> trajectory dict, driven exactly as
    Sim.__gen_data_from_pathgen does (ins_sim.py:444-472): parse (ins_sim.py:578-640), then
    path_gen -- here the host-side restatement in csrc/pathgen_host.h (pathgen.py), ~200x faster
    than the reference's Python loop and identical to it to the last bits."""
    from . import pathgen
    ini_pva, cmd = pathgen.parse_motion(motion_def)
    mobility = pathgen.parse_mode(mode)
    output_def = np.array([[1.0, fs], [1.0 if gps else -1.0, fs_gps if gps else fs],
                           [1.0 if odo else -1.0, fs]])
    rtn = pathgen.path_gen(ini_pva, cmd, output_def, mobility, ref_frame, magnetometer, wmm_file, wmm_date)
    out = {'time': rtn['nav'][:, 0] / fs, 'ref_pos': np.ascontiguousarray(rtn['nav'][:, 1:4]),
           'ref_vel': np.ascontiguousarray(rtn['nav'][:, 4:7]),
           'ref_att': np.ascontiguousarray(rtn['nav'][:, 7:10]),
           'ref_accel': np.ascontiguousarray(rtn['imu'][:, 1:4]),
           'ref_gyro': np.ascontiguousarray(rtn['imu'][:, 4:7]), 'ini': ini_pva}
    if odo:
        out['ref_odo'] = np.ascontiguousarray(rtn['odo'][:, 2])
    if magnetometer:
        out['ref_mag'] = np.ascontiguousarray(rtn['mag'][:, 1:4])
    if gps:
        out['gps_time'] = rtn['gps'][:, 0] / fs
        out['ref_gps'] = np.ascontiguousarray(rtn['gps'][:, 1:7])
        out['gps_visibility'] = np.ascontiguousarray(rtn['gps'][:, 7])
    return out


class _DataDict(dict):
    """Sim.data: a dict whose values may be registered as thunks and are built on first read."""

    class _Thunk:
        def __init__(self, fn):
            self.fn = fn

    def defer(self, key, fn):
        dict.__setitem__(self, key, _DataDict._Thunk(fn))

    def __getitem__(self, key):
        v = dict.__getitem__(self, key)
        if isinstance(v, _DataDict._Thunk):
            v = v.fn()
            dict.__setitem__(self, key, v)
        return v

    def get(self, key, default=None):
        return self[key] if key in self else default


def _gather_allan(curves, noise, total):
    """Every rank's Allan results in one gather: its curves [R_local, L, 6] and, with the fit, its noise terms
    [R_local, 6, 6] (None without) go as rows [R_local, 6 L (+ 36)].  Returns ([total, L, 6], [total, 6, 6] or
    None) in run order on every rank."""
    R, L = curves.shape[0], curves.shape[1]
    rows = curves.reshape(R, L * 6)
    if noise is not None:
        rows = np.concatenate([rows, noise.reshape(R, 36)], axis=1)
    rows = dist.gather_rows(torch.from_numpy(np.ascontiguousarray(rows)), total)
    return (rows[:, :L * 6].reshape(total, L, 6),
            None if noise is None else rows[:, L * 6:].reshape(total, 6, 6))


def _keyed(name, per_run):
    """{'<name>_<r>': per_run[r]}: an algorithm's per-run outputs under the reference's run keys."""
    return {'%s_%d' % (name, r): v for r, v in enumerate(per_run)}


class _LazyDevice(dict):
    """The trajectory on the device, each array uploaded when first asked for: ref_gyro, ref_accel, ref_odo,
    ref_gps, ref_mag, ref_nav ([n][9] att, pos, vel), and for the filter gps_idx (the IMU sample of each GPS
    row) and gps_vis (visibility).  The single-GPU run() goes through a plan that stages the host arrays
    itself; the Allan path never needs the navigation rows."""

    def __init__(self, sim):
        super().__init__()
        self._sim = weakref.ref(sim)     # no reference cycle: a Sim is freed (with its device arrays) when dropped

    def __missing__(self, key):
        sim = self._sim()
        t = sim._traj
        if key == 'gps_idx':
            self[key] = torch.from_numpy(np.rint(np.asarray(t['gps_time']) * sim.fs[0]).astype(np.int64)).cuda()
        elif key == 'ref_nav':
            self[key] = engine.to_device(np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1))
        else:
            self[key] = engine.to_device(t['gps_visibility' if key == 'gps_vis' else key])
        return self[key]


class LazyRuns(Mapping):
    """dict-like {key: (n,3) array} of per-run histories, materialised on first access by
    re-running the requested runs with history output (deterministic Philox streams).
    Keys are the reference's: the run index for sensor data (prefix None), '<algo>_<run>' for
    algorithm outputs.  Nothing is built per run until somebody asks (a Monte-Carlo
    experiment with 10^5 runs must not spend its time making 10^5 Python strings)."""

    def __init__(self, sim, name, count, prefix=None):
        # a weak reference: Sim.data -> LazyRuns -> Sim would be a cycle that only the cyclic collector frees,
        # and a Sim owns device and pinned buffers
        self._sim_ref, self._name, self._count, self._prefix = weakref.ref(sim), name, int(count), prefix

    @property
    def _sim(self):
        sim = self._sim_ref()
        if sim is None:
            raise ReferenceError('the Sim these run histories belong to no longer exists')
        return sim

    def _key(self, r):
        return r if self._prefix is None else '%s_%d' % (self._prefix, r)

    def _run_of(self, key):
        if self._prefix is None:
            r = key
        else:
            if not isinstance(key, str) or not key.startswith(self._prefix + '_'):
                raise KeyError(key)
            try:
                r = int(key[len(self._prefix) + 1:])
            except ValueError:
                raise KeyError(key)
        if not isinstance(r, (int, np.integer)) or not 0 <= r < self._count:
            raise KeyError(key)
        return int(r)

    def __contains__(self, key):
        try:
            self._run_of(key)
            return True
        except KeyError:
            return False

    def __iter__(self):
        return (self._key(r) for r in range(self._count))

    def __len__(self):
        return self._count

    def __getitem__(self, key):
        return self._sim._history(self._name, self._run_of(key))


# ------------------------------------------------------------------ the facade --
_UNITS = {  # name -> (description, units, output units)   ins_data_manager.py:85-216
    'att_euler': ('simulation attitude (Euler, ZYX)  from algo', ['rad'] * 3, ['deg'] * 3),
    'pos': ('simulation position from algo', ['rad', 'rad', 'm'], ['deg', 'deg', 'm']),
    'vel': ('simulation velocity from algo', ['m/s'] * 3, ['m/s'] * 3),
}


_SENSOR_UNITS = {  # sensor data with a ref_ counterpart -> (units, output units), ins_data_manager.py:96-143
    'gyro': (['rad/s'] * 3, ['deg/s'] * 3),
    'accel': (['m/s^2'] * 3, ['m/s^2'] * 3),
    'mag': (['uT'] * 3, ['uT'] * 3),
    'gps': (['rad', 'rad', 'm', 'm/s', 'm/s', 'm/s'], ['deg', 'deg', 'm', 'm/s', 'm/s', 'm/s']),
}
_REF_OF = {'att_euler': 'ref_att', 'pos': 'ref_pos', 'vel': 'ref_vel'}   # trajectory key of an output's truth
_MAGCAL_UNITS = {'soft_iron': ['-'] * 9, 'hard_iron': ['uT'] * 4}   # MagCal calibration errors


def _first_at(t, start_s):
    """Index of the first time >= start_s; past the end: the reference's message and 0
    (ins_data_manager.py:774-782)."""
    idx = np.where(np.asarray(t) >= start_s)[0]
    if idx.shape[0] == 0:
        print('err_stats_start exceeds max data points.')
        return 0
    return int(idx[0])


def _host_stats(e):
    """InsDataMgr.__array_stats (ins_data_manager.py:797-808) over axis 0."""
    return np.stack([np.max(np.abs(e), 0), np.average(e, 0), np.std(e, 0)])


class Sim(object):
    '''
    INS Monte-Carlo simulation engine (device-backed).
    '''

    def __init__(self, fs, motion_def, ref_frame=0, imu=None, mode=None, env=None,
                 algorithm=None, seed=0, lanes_per_run=0, history_block=32, run_base=0,
                 wmm_file=None, wmm_date=None):
        '''
        Args: as gnss_ins_sim.sim.ins_sim.Sim (ins_sim.py:31-124), plus
            seed: Philox key of the experiment (the reference is unseeded; here every
                (seed, run) pair names one reproducible noise realisation).
            lanes_per_run: CUDA lane-group width (0 = automatic).
            history_block: runs materialised together on a lazy history access.
            run_base: Philox stream id of run 0 (run r draws stream run_base + r), so that
                separate experiments can extend one ensemble without reusing streams.
            wmm_file: World Magnetic Model coefficients (NOAA .COF) for a 9-axis IMU on a motion
                definition; default: geoparams/WMM.COF of an installed gnss_ins_sim package.
            wmm_date: datetime.date the field is evaluated at (default: today, as the reference).
        '''
        self.fs = list(fs) if isinstance(fs, (list, tuple, np.ndarray)) else [float(fs), 0.0, 0.0]
        self.imu = imu
        self.mode = mode
        self.env = env
        self.ref_frame = ref_frame if ref_frame in (0, 1) else 0
        self.seed = int(seed)
        self.lanes_per_run = int(lanes_per_run)
        self.history_block = int(history_block)
        self._force_fed = False    # tests: run free integration as K1 then K2 even without the IMU's extra terms
        self.run_base = int(run_base)
        self.wmm_file, self.wmm_date = wmm_file, wmm_date
        self.data_src = motion_def
        self.sim_count = 1
        self.sim_complete = False
        self.sim_results = False
        self.sum = ''
        self.algo = algorithm
        if algorithm is not None and not isinstance(algorithm, (list, tuple)):
            self.algo = [algorithm]
        if self.algo is not None:
            for a in self.algo:   # InsAlgoMgr.__check_algo, ins_algo_manager.py:116-127
                try:
                    ok = len(a.input) >= 1 and len(a.output) >= 1
                except Exception:
                    ok = False
                if not ok:
                    raise ValueError('algorithm input or output is not a valid list or tuple.')
        self.data = _DataDict()  # name -> ndarray | dict-of-runs | LazyRuns (| thunk, until first read)
        self.err_stats = {}     # end-point ensemble statistics of the last run()
        self._traj = None
        self._logged = None      # data read from a logged-data directory (no sensor model)
        self._dev = None         # _LazyDevice of the trajectory

    # ---- names ------------------------------------------------------------
    def algo_name(self, i):
        """InsAlgoMgr.get_algo_name, ins_algo_manager.py:98-114"""
        a = self.algo[i]
        return a.name if hasattr(a, 'name') else 'algo' + str(i)

    # ---- trajectory -------------------------------------------------------
    def _load_trajectory(self):
        src = self.data_src
        if isinstance(src, dict) or (isinstance(src, str) and src.endswith('.npz')):
            traj = load_trajectory(src)
        elif isinstance(src, str):
            if os.path.isdir(src):
                self._load_logged(src)
                return
            traj = trajectory_from_motion_def(self.fs[0], src, self.ref_frame, self.mode,
                                              bool(self.imu and self.imu.magnetometer),
                                              bool(self.imu and self.imu.odo),
                                              bool(self.imu and self.imu.gps) and self.fs[1] > 0,
                                              self.fs[1], self.wmm_file, self.wmm_date)
        else:
            raise TypeError('motion_def must be a trajectory dict, an .npz path or a motion '
                            'definition csv/string')
        n = traj['ref_gyro'].shape[0]
        if 'time' not in traj:
            traj['time'] = np.arange(n) / self.fs[0]
        self._traj = traj
        d = self.data
        d['fs'], d['ref_frame'], d['time'] = self.fs[0], self.ref_frame, traj['time']
        d['ref_pos'], d['ref_vel'], d['ref_att_euler'] = traj['ref_pos'], traj['ref_vel'], traj['ref_att']
        d['ref_accel'], d['ref_gyro'] = traj['ref_accel'], traj['ref_gyro']
        d.defer('ref_att_quat', lambda: euler2quat_zyx(traj['ref_att']))   # built when first read
        for k in ('ref_odo', 'gps_time', 'ref_gps', 'gps_visibility', 'ref_mag'):
            if k in traj:
                d[k] = traj[k]
        self._nav_end = np.concatenate([traj['ref_att'][-1], traj['ref_pos'][-1], traj['ref_vel'][-1]])
        self._dev = _LazyDevice(self)

    # ---- run ----------------------------------------------------------------
    def run(self, num_times=1):
        '''
        run simulation.
        Args:
            num_times: run the simulation for num_times times with given IMU error model.
        '''
        self.sim_count = max(int(num_times), 1)
        if self._traj is None and self._logged is None:
            self._load_trajectory()
        if self._logged is not None:
            return self._run_logged()
        if self.imu is None:
            raise ValueError('imu must be an IMU model when data are generated from a trajectory')
        terms = self._imu_terms()
        for a in self.algo or []:       # refused before anything of the Sim is reset
            if terms and isinstance(a, FreeIntegrationOdo):
                raise ValueError('%s generates its IMU inside its kernel, which makes no quantisation, rate '
                                 'random walk, rate ramp or run-to-run bias, scale-factor or misalignment error: '
                                 'the IMU sets %s' % (type(a).__name__, terms))
            # K7 draws the turn-on bias; its 15 states have no place for the rest
            rest = [t for t in terms if not t.endswith(' b_std')]
            if rest and isinstance(a, InsLoose):
                raise ValueError('%s generates its IMU inside its kernel, which makes no quantisation, rate '
                                 'random walk, rate ramp or run-to-run scale-factor or misalignment error: '
                                 'the IMU sets %s' % (type(a).__name__, rest))
        self._blocks = {}        # (block, name) -> [runs of the block, ...] host histories (_history)
        self._proc = {}          # (algo index, start [s], position frame) -> [R, 3, 9] process statistics
        self._sens = {}          # (source, first row) -> sensor error statistics (_sensor_launch)
        self._all_hist = None    # (algo index, first run, arrays) of the last histories() with stride 1
        self.err_stats = {}
        self._mc = {}
        self._magcal = {}        # algo index -> [3, 13] statistics of the calibration errors (MagCal)
        self._vib_acc = parse_env(self.env['acc'], self.fs[0]) if self.env and 'acc' in self.env else None
        self._vib_gyro = parse_env(self.env['gyro'], self.fs[0]) if self.env and 'gyro' in self.env else None
        self._psd_cache = {}
        R = self.sim_count
        if getattr(self.imu, 'magnetometer', False) and 'ref_mag' not in self._traj:
            raise ValueError('imu has a magnetometer (axis=9) but the trajectory has no ref_mag')
        self._shard = dist.shard(R)
        for a in self.algo or []:      # outputs start afresh: a _Merged view holds the plugins of this run only
            for o in a.output:
                self.data.pop(o, None)
        self.data['accel'] = LazyRuns(self, 'accel', R)
        self.data['gyro'] = LazyRuns(self, 'gyro', R)
        if getattr(self.imu, 'odo', False):
            if 'ref_odo' not in self._traj:
                raise ValueError('imu.odo is on but the trajectory has no ref_odo')
            self.data['odo'] = LazyRuns(self, 'odo', R)
        if getattr(self.imu, 'gps', False) and 'ref_gps' in self._traj:
            self.data['gps'] = LazyRuns(self, 'gps', R)     # pathgen.gps_gen per run (ins_sim.py:497-500)
        if getattr(self.imu, 'magnetometer', False):
            self.data['mag'] = LazyRuns(self, 'mag', R)     # pathgen.mag_gen per run (ins_sim.py:501-503)
        if self.algo is not None:
            for i, a in enumerate(self.algo):
                if isinstance(a, FreeIntegration):     # incl. the odometer variant
                    self._run_free_integration(i, a)
                elif isinstance(a, SeriesEstimator):
                    self._run_allan(i, a)
                elif isinstance(a, InsLoose):
                    self._run_ins_loose(i, a)
                elif isinstance(a, MagCal):
                    self._run_magcal(i, a)
                else:
                    self._run_plugin(i, a, self._generated_inputs)
        self.sim_complete = True

    # ---- logged data (ins_sim.py:415-451: data from files instead of pathgen) -------------------
    def _load_logged(self, path):
        """Every supported .csv of the directory in internal units; no sensor model is applied."""
        d = logged.read_data_dir(os.path.abspath(path), self.ref_frame)
        if 'time' not in d:
            for v in d.values():
                a = next(iter(v.values())) if isinstance(v, dict) else v
                d['time'] = np.arange(a.shape[0]) / self.fs[0]
                break
        self._logged = d
        self.data.update(d)
        self.data['fs'], self.data['ref_frame'] = self.fs[0], self.ref_frame
        if 'ref_att_euler' in d and 'ref_att_quat' not in d:
            self.data.defer('ref_att_quat', lambda: euler2quat_zyx(d['ref_att_euler']))
        # what the error statistics need of a trajectory
        self._traj = {k2: d[k1] for k1, k2 in (('ref_pos', 'ref_pos'), ('ref_vel', 'ref_vel'),
                                               ('ref_att_euler', 'ref_att'), ('time', 'time')) if k1 in d}

    def _logged_sets(self, name):
        """[R, n, ...] stack of the first sim_count sets (keys 0 .. R-1) of a per-run quantity."""
        sets = self._logged.get(name)
        if not isinstance(sets, dict):
            raise ValueError('the data directory holds no %s-<key>.csv' % name)
        try:
            return np.stack([sets[r] for r in range(self.sim_count)])
        except KeyError as e:
            raise ValueError('the data directory holds no %s-%s.csv' % (name, e.args[0]))

    def _run_logged(self):
        """Algorithms on the logged sets 0 .. sim_count-1 (InsAlgoMgr.run_algo over the keys,
        ins_algo_manager.py:73-95): one batched launch per algorithm, outputs keyed
        '<algo>_<key>'; end-point error statistics if the directory has the reference files."""
        self._proc, self.err_stats, self._mc, self._sens, self._magcal = {}, {}, {}, {}, {}
        self._shard = (0, self.sim_count)
        d = self._logged
        for i, a in enumerate(self.algo or []):
            name = self.algo_name(i)
            if isinstance(a, FreeIntegration):
                self._mc[i] = {'base': a.run_times, 'end_err': None}
                if isinstance(a, FreeIntegrationOdo):
                    att, pos, vel = a.run_batch(self.ref_frame, self.fs[0], self._logged_sets('gyro'),
                                                self._logged_sets('odo'))
                else:
                    att, pos, vel = a.run_batch(self.ref_frame, self.fs[0], self._logged_sets('gyro'),
                                                self._logged_sets('accel'))
                for out, arr in (('att_euler', att), ('pos', pos), ('vel', vel)):
                    self.data[out] = dict(self.data[out]) if isinstance(self.data.get(out), dict) else {}
                    self.data[out].update(_keyed(name, arr))
                self.data['att_quat'] = DerivedRuns(self.data['att_euler'], euler2quat_zyx)
                if all(k in d for k in ('ref_att_euler', 'ref_pos', 'ref_vel')):
                    err = np.concatenate([
                        (att[:, -1] - d['ref_att_euler'][-1] + math.pi) % (2.0 * math.pi) - math.pi,
                        pos[:, -1] - d['ref_pos'][-1], vel[:, -1] - d['ref_vel'][-1]], axis=1)
                    self._mc[i]['end_err'] = err
                    self.err_stats[name] = engine.error_stats(engine.to_device(err)).cpu().numpy()
            elif isinstance(a, SeriesEstimator):
                self._publish_allan(name, a, *a.run_batch(self.fs[0], self._logged_sets('accel'),
                                                          self._logged_sets('gyro')))
            elif isinstance(a, InsLoose):
                self._run_logged_ins_loose(i, a)
            elif isinstance(a, MagCal):
                si, hi, cal = a.run_batch(self._logged_sets('mag'))
                self._publish_magcal(name, si, hi)
                self.data['mag_cal'] = _keyed(name, cal)
            else:
                self._run_plugin(i, a, self._logged_inputs)
        self.sim_complete = True

    def _run_logged_ins_loose(self, i, algo):
        """The filter on the logged sets gyro-k, accel-k, gps-k (k < sim_count) with gps_time and, if present,
        gps_visibility.  Model: algo.imu, else the Sim's imu.  Initial state: algo.ini, else the first reference
        row (velocity rotated to the body frame), plus the initial-covariance draw of run run_base + k under the
        Sim's seed, as the generated experiment draws it: a directory save_data wrote from a generated filter
        experiment filters back to that experiment.  Run blocks are sized to the free device memory (inputs and
        histories: 168 B per run-sample).  End-point errors and their statistics if the reference files exist.
        With InsLoose(align_yaw=...) every run initialises itself from its measurements: no initial state, no
        draw, and no reference files needed."""
        d, name, R = self._logged, self.algo_name(i), self.sim_count
        if self.ref_frame != 0:
            raise ValueError('ins_loose works in ref_frame 0 (LLA positions, NED velocities)')
        imu = algo.model(self.imu)
        has_ref = all(k in d for k in ('ref_att_euler', 'ref_pos', 'ref_vel'))
        ini = algo.ini
        if ini is None and algo.align_yaw is None:
            if not has_ref:
                raise ValueError('InsLoose on a data directory needs ini_pos_vel_att or the ref_pos, ref_vel and '
                                 'ref_att_euler files')
            att = d['ref_att_euler'][0]
            ini = np.concatenate([d['ref_pos'][0], euler2dcm_zyx(att).dot(d['ref_vel'][0]), att])
        if 'gps_time' not in d:
            raise ValueError('the data directory holds no gps_time.csv')
        gyro, accel, gps = (self._logged_sets(k) for k in ('gyro', 'accel', 'gps'))
        vis = d.get('gps_visibility')
        vis = np.ones(len(d['gps_time'])) if vis is None else vis
        gps_idx = gps_sample_index(self.fs[0], d['time'], d['gps_time'])
        ref_nav = engine.to_device(np.concatenate([d['ref_att_euler'], d['ref_pos'], d['ref_vel']], axis=1)) \
            if has_ref else None
        outs = {o: [] for o in ('pos', 'vel', 'att_euler', 'wb', 'ab')}
        errs, bias, start = [], [], 0
        block = self._allan_block(168, 3)
        for r0 in range(0, R, block):
            r1 = min(R, r0 + block)
            res = algo.launch(self.fs[0], engine.to_device(gyro[r0:r1]), engine.to_device(accel[r0:r1]),
                              engine.to_device(gps[r0:r1]), gps_idx, vis, imu, ini, self.seed, True,
                              self.run_base + r0, ref_nav)
            start = res.start
            for o, t in zip(outs, (res.pos, res.vel, res.att, res.wb, res.ab)):
                outs[o].append(t.cpu().numpy())
            bias.append(res.end_bias.cpu().numpy())
            if has_ref:
                errs.append(res.end_err.cpu().numpy())
            del res
        algo.run_times += R
        for o, parts in outs.items():
            self.data[o] = dict(self.data[o]) if isinstance(self.data.get(o), dict) else {}
            self.data[o].update(_keyed(name, np.concatenate(parts)))
        self._mc[i] = {'base': 0, 'end_err': np.concatenate(errs) if has_ref else None,
                       'end_bias': np.concatenate(bias), 'start': start if R else 0}
        if has_ref:
            self.err_stats[name] = engine.error_stats(engine.to_device(self._mc[i]['end_err'])).cpu().numpy()

    def _logged_inputs(self, algo, r):
        """Inputs of run r of a foreign plugin on logged data: set r of per-run data, everything else as is."""
        args = []
        for nm in algo.input:
            v = self.data.get(nm)
            if isinstance(v, dict):
                v = v.get(r)
            if v is None:
                raise ValueError('algorithm input %r is not in the data directory' % nm)
            args.append(v)
        return args

    def _run_plugin(self, i, algo, inputs):
        """A reference-style plugin run on the host (the per-run protocol of InsAlgoMgr.run_algo,
        ins_algo_manager.py:73-95); inputs(algo, r): its input list for run r."""
        name = self.algo_name(i)
        outs = {o: {} for o in algo.output}
        for r in range(self.sim_count):
            args = inputs(algo, r)
            algo.reset()
            algo.run(copy.deepcopy(args))
            for o, v in zip(algo.output, algo.get_results()):
                outs[o]['%s_%d' % (name, r)] = v
        self.data.update(outs)

    def _mc_config(self, ai, r0, runs, **kw):
        """Config for experiment runs [r0, r0+runs) of algorithm ai; kw: make_mc_config's stats_start,
        dump_runs, dump_stride, proc_pos_frame.  Philox streams are named by the experiment run index (all
        algorithms see the same sensor data, as in the reference where loop A runs once); the
        initial-state rule counts the plugin's own run_times."""
        algo = self.algo[ai]
        n = self._traj['ref_gyro'].shape[0]
        vib_gyro, vib_acc = self._vib_pair(runs, r0)
        return engine.make_mc_config(
            self.ref_frame, self.fs[0], n, runs, self.seed, self.imu.gyro_err, self.imu.accel_err,
            algo.ini_sets.shape[0], algo.ini_sets.shape[1], earth_rot=algo.earth_rot,
            run_offset=self.run_base + r0, ini_offset=self._mc[ai]['base'] + r0,
            vib_gyro=vib_gyro, vib_accel=vib_acc,
            lanes_per_run=self.lanes_per_run or algo.lanes_per_run, **kw, **self._odo_args(algo))

    def _mc_launch(self, ai, r0, runs, stats_start=-1, dump_runs=0, dump_stride=1, proc_pos_frame=0, **kw):
        """K12 for experiment runs [r0, r0+runs) of algorithm ai on the device trajectory; kw: what
        engine.mc_free_integration outputs beside the end-point errors."""
        cfg = self._mc_config(ai, r0, runs, stats_start=stats_start, dump_runs=dump_runs, dump_stride=dump_stride,
                              proc_pos_frame=proc_pos_frame)
        d = self._dev
        return engine.mc_free_integration(cfg, d['ref_gyro'], d['ref_accel'], d['ref_nav'],
                                          self.algo[ai].ini_device(), **kw)

    def _odo_args(self, algo):
        """Odometer variant: noise model (imu.odo_err) and the true forward speed on the device."""
        if not isinstance(algo, FreeIntegrationOdo):
            return {}
        if not getattr(self.imu, 'odo', False) or 'ref_odo' not in self._traj:
            raise ValueError('free_integration_odo needs IMU(odo=True) and a trajectory with ref_odo')
        return {'odo_err': self.imu.odo_err, 'ref_odo': self._dev['ref_odo']}

    def _vib_pair(self, runs, r0):
        """(vib_gyro, vib_accel) arguments for experiment runs [r0, r0+runs): parsed dicts, or
        for the PSD model a VIB_SERIES over device series made by K5 for exactly those runs
        (time_series_from_psd is called per run and axis, pathgen.py:478-485, :541-548)."""
        out = []
        for sensor, v in ((1, self._vib_gyro), (0, self._vib_acc)):
            if v is not None and v['type'] == 'psd':
                key = (sensor, runs, r0)
                if key not in self._psd_cache:
                    n = self._traj['ref_gyro'].shape[0]
                    if len(self._psd_cache) > 8:    # evict, but never a series of THIS (runs, r0) block:
                        for k in [k for k in self._psd_cache if k[1:] != (runs, r0)]:   # its Vib is in use
                            del self._psd_cache[k]
                    self._psd_cache[key] = engine.psd_series(self.fs[0], n, runs, sensor, v, self.seed,
                                                             self.run_base + r0)
                series, N = self._psd_cache[key]
                out.append(engine.vib_series(series, N))   # the Vib keeps its series tensor alive
            else:
                out.append(v)
        return out[0], out[1]

    def _uses_psd(self):
        return any(v is not None and v['type'] == 'psd' for v in (self._vib_acc, self._vib_gyro))

    def _imu_terms(self):
        """The IEEE Std 952 terms and run-to-run errors the IMU sets (non-zero 'q', 'rrw', 'rr', 'b_std', 'sf',
        'ma'), e.g. ['gyro rrw', 'gyro sf']; [] for none.  Only K1 and K9 make them."""
        return ['%s %s' % (s, k) for s, err in (('gyro', self.imu.gyro_err), ('accel', self.imu.accel_err))
                for k in _lib.set_terms(err) + _lib.set_run_errors(err)]

    def imu_run_errors(self):
        """The run-to-run errors every run of the experiment draws: {'accel': [R, 3, 4], 'gyro': [R, 3, 4]} (numpy;
        R = the runs of the last run(), all ranks' runs), row i = (S[i][0], S[i][1], S[i][2], b_run[i]): the run's
        measurement is the truth plus b_run + S truth plus everything else the IMU model makes.  Computed on the
        device from the global run ids (run_base + r) and the seed, so every rank gets the same table.  All zero for
        an IMU without 'b_std', 'sf' or 'ma'."""
        if self.imu is None:
            raise ValueError('imu_run_errors needs an IMU model')
        t = engine.imu_run_errors(self.sim_count, self.imu.gyro_err, self.imu.accel_err, self.seed,
                                  run_offset=self.run_base).cpu().numpy()
        return {'accel': t[:, 0], 'gyro': t[:, 1]}

    def _fed(self, ai):
        """True if free-integration plugin ai runs as K1 then K2 on the materialised series (the IMU has terms
        K12's generator does not make) instead of K12."""
        return not isinstance(self.algo[ai], FreeIntegrationOdo) and (self._force_fed or bool(self._imu_terms()))

    def _fed_blocks(self, ai, lo, hi):
        """K1 (with the IMU's terms) then K2 for experiment runs [lo, hi) of free-integration plugin ai, in run
        blocks sized to the free device memory (120 B per run-sample: the series and the histories): yields
        (r0, att, pos, vel, gyro, accel), CUDA [runs, n, 3].  Philox makes a block's rerun identical."""
        algo = self.algo[ai]
        block = max(1, min(hi - lo, self._allan_block(120, 3)))
        for r0 in range(lo, hi, block):
            r1 = min(hi, r0 + block)
            gyro, accel = self._noise_block(r0, r1)
            att, pos, vel = engine.free_integration(self.ref_frame, self.fs[0], gyro, accel, algo.ini_device(),
                                                    earth_rot=algo.earth_rot,
                                                    run_offset=self._mc[ai]['base'] + r0)
            yield r0, att, pos, vel, gyro, accel
            del att, pos, vel, gyro, accel

    def _fed_errors(self, att, pos, vel, frame=0, rows=slice(None)):
        """[runs, rows, 9] host errors of K2 history rows against the trajectory's: attitude wrapped to [-pi, pi),
        position in the frame's units (engine.POS_FRAME_*), velocity."""
        ref = {k: self._traj[k][rows] for k in ('ref_att', 'ref_pos', 'ref_vel')}
        ea = (att[:, rows].cpu().numpy() - ref['ref_att'][None] + math.pi) % (2.0 * math.pi) - math.pi
        x = pos[:, rows].cpu().numpy()
        ep = np.stack([lla_error_metres(xr, ref['ref_pos'], frame) for xr in x]) if frame else x - ref['ref_pos'][None]
        return np.concatenate([ea, ep, vel[:, rows].cpu().numpy() - ref['ref_vel'][None]], axis=2)

    def _run_free_integration(self, i, algo):
        name = self.algo_name(i)
        lo, hi = self._shard
        self._mc[i] = {'base': algo.run_times, 'end_err': None}   # plugin's run counter at run 0
        err, stats = np.zeros((0, 9)), np.zeros((3, 9))
        if self._fed(i):
            if hi > lo:
                err = np.concatenate([self._fed_errors(a, p, v, rows=slice(-1, None))[:, 0]
                                      for _, a, p, v, _, _ in self._fed_blocks(i, lo, hi)])
                stats = engine.error_stats(engine.to_device(err)).cpu().numpy()
            self._mc[i]['end_err'] = err
            self.err_stats[name] = dist.combine_local_stats(stats, hi - lo)
        elif not isinstance(algo, FreeIntegrationOdo):
            # the plan path on this rank's shard (pinned staging, one H2D, K12, K3, one D2H);
            # with several ranks the [3][9] shard statistics are merged by one all_gather
            # the exchange path is chosen from the LARGEST shard, a rank-independent quantity (shards
            # differ by one run; every rank must take the same collective)
            w = dist.world()
            p2p = dist.fused_exchange(9) if w > 1 and -(-self.sim_count // w) * 9 <= (1 << 17) else None
            plan = None
            if hi > lo:
                cfg = self._mc_config(i, lo, hi - lo)
                t = self._traj
                plan = engine.get_plan(cfg.n, cfg.runs, cfg.ini_sets, cfg.ini_rows)
                if self._uses_psd():
                    # K5 wrote the vibration series on torch's current stream; the plan runs K12 on
                    # its own non-blocking stream: order the two
                    torch.cuda.current_stream().synchronize()
                err, stats = plan.run(cfg, t['ref_gyro'], t['ref_accel'], self._nav_end, algo.ini_sets,
                                      want_stats=p2p is None)
            self._mc[i]['end_err'] = err
            if p2p is not None:
                # K3x on the plan's device buffer: statistics + NVLink exchange + merge, one kernel
                # (plan.run has synchronised: the errors are final; torch's stream orders the copy)
                merged = p2p(plan.err_device_ptr() if plan else None, hi - lo).cpu().numpy().copy()
                if p2p.timed_out():      # a peer never arrived: the merge is incomplete, never use it
                    p2p.reset_timeout()
                    raise RuntimeError('statistics exchange (K3x) timed out waiting for a peer rank; '
                                       'the ensemble statistics of this run() are not available')
                self.err_stats[name] = merged
            else:
                self.err_stats[name] = dist.combine_local_stats(stats, hi - lo)
        else:
            if hi > lo:
                res = self._mc_launch(i, lo, hi - lo)
                stats = engine.error_stats(res.end_err).cpu().numpy()
                err = res.end_err.cpu().numpy()
            self._mc[i]['end_err'] = err
            self.err_stats[name] = dist.combine_local_stats(stats, hi - lo)
        algo.run_times += self.sim_count
        for out in ('att_euler', 'pos', 'vel'):     # several free-integration plugins: one view over all
            prev = self.data.get(out)
            lazy = LazyRuns(self, (i, out), self.sim_count, prefix=name)
            if isinstance(prev, _Merged):
                prev.add(lazy)
            elif isinstance(prev, LazyRuns):
                self.data[out] = _Merged([prev, lazy])
            else:
                self.data[out] = lazy
        self.data['att_quat'] = DerivedRuns(self.data['att_euler'], euler2quat_zyx)

    def _noise_block(self, r0, r1, layout=engine.LAYOUT_RUN_MAJOR):
        """K1 for global-in-experiment runs [r0, r1): CUDA gyro, accel [r1-r0, n, 3]
        ([r1-r0, 3, n] with LAYOUT_CHANNEL_MAJOR)."""
        d = self._dev
        vib_gyro, vib_acc = self._vib_pair(r1 - r0, r0)
        return engine.imu_noise(self.fs[0], r1 - r0, d['ref_gyro'], d['ref_accel'],
                                self.imu.gyro_err, self.imu.accel_err, self.seed,
                                run_offset=self.run_base + r0, vib_gyro=vib_gyro,
                                vib_accel=vib_acc, layout=layout)

    def _generated_inputs(self, algo, r):
        """Inputs of run r of a foreign plugin: gyro and accel from K1 (one launch per run), mag from the
        history block get_data(['mag']) serves, everything else from self.data."""
        gyro, accel = self._noise_block(r, r + 1)
        per_run = {'gyro': gyro[0].cpu().numpy(), 'accel': accel[0].cpu().numpy()}
        if 'mag' in algo.input and 'mag' in self.data:
            per_run['mag'] = self.data['mag'][r]
        args = []
        for nm in algo.input:
            v = per_run[nm] if nm in per_run else self.data.get(nm)
            if v is None or isinstance(v, Mapping):
                raise ValueError('algorithm input %r is not generated by this engine' % nm)
            args.append(v)
        return args

    # ---- Allan variance (K1 + K4, or K1 fused into K4) ------------------------------------------
    def _allan_block(self, bytes_per_sample, share):
        """Runs per Allan block of this rank's shard: `bytes_per_sample` of device memory per run-sample, in
        at most 1/share of the free device memory (free on the device + cached by torch's allocator but
        unused)."""
        lo, hi = self._shard
        n = len(self.data['time'])
        if torch.cuda.is_available():
            free_b = (torch.cuda.mem_get_info()[0] + torch.cuda.memory_reserved()
                      - torch.cuda.memory_allocated())
        else:
            free_b = 2 ** 31
        return max(1, min(max(hi - lo, 1), int(free_b / share // (n * bytes_per_sample)) or 1))

    def _publish_allan(self, name, algo, tau, accel, gyro, *per_series):
        """The plugin's first output, its abscissa (algo_time: the same tau for every run; algo_freq for Psd),
        and its accel and gyro outputs [R, ntau, 3] (ad_* for Allan, hd_* for Hadamard, psd_* for Psd) under run
        keys, then its per-series outputs in output order (Allan(fit=True): noise_accel, noise_gyro [R, 3, 6]).
        Plugins of one Sim with the same abscissa share it: each replaces its own run keys in it and keeps the
        others'."""
        t, o_accel, o_gyro, *o_rest = algo.output
        prev = self.data.get(t)
        keep = {k: v for k, v in prev.items() if not k.startswith(name + '_')} if isinstance(prev, dict) else {}
        self.data[t] = dict(keep, **_keyed(name, [tau] * len(accel)))
        self.data[o_accel] = _keyed(name, accel)
        self.data[o_gyro] = _keyed(name, gyro)
        for o, v in zip(o_rest, per_series):
            self.data[o] = _keyed(name, v)

    def _run_allan(self, i, algo):
        """The Allan deviations of this rank's shard of the runs, in run blocks sized to the free device
        memory; the [R, ntau, 6] deviations of all ranks are gathered (a few hundred KB).  Without a vibration
        model and with series longer than one chunk, K1 is fused into K4's first level (engine.allan_mc) and
        the only device memory is the decade-sum workspace (about 2 B per run-sample), so run blocks are
        rarely needed; otherwise K1 materialises the series (48 B per run-sample) for K4 (~2 B of workspace).
        Allan(overlapping=True) and Hadamard() always materialise: K4o needs its prefix workspace (about 48 B per
        run-sample for the three series of one sensor) beside the series.  Psd() materialises too, with K11's
        chunk sums beside the series; its abscissa is the frequency grid instead of tau.  Allan(fit=True) fits
        every block's curves on the device (K13, engine.allan_fit) before they are copied back; the [R, 6, 6]
        noise terms (channels accel x y z, gyro x y z) are gathered with the curves."""
        lo, hi = self._shard
        n = self._traj['ref_gyro'].shape[0]
        fused = (algo.fused and self._vib_acc is None and self._vib_gyro is None and n > 5040
                 and not self._imu_terms() and os.environ.get('B2INS_ALLAN_FUSED', '1') != '0')
        fit = getattr(algo, 'fit', False)
        tau = algo.abscissa(n, self.fs[0])
        block = self._allan_block(6 * 2, 2) if fused else self._allan_block(algo.run_bytes(n), 3)
        parts, fits = [], []      # [runs, ntau, 6]: accel, gyro; [runs, 6, 6]: the noise terms of each channel
        for r0 in range(lo, hi, block):
            r1 = min(hi, r0 + block)
            if fused:
                d = self._dev
                avar, _ = engine.allan_mc(self.fs[0], r1 - r0, d['ref_gyro'], d['ref_accel'], self.imu.gyro_err,
                                          self.imu.accel_err, self.seed, run_offset=self.run_base + r0)
                if fit:
                    fits.append(engine.allan_fit(self.fs[0], n, avar).reshape(r1 - r0, 6, 6).cpu().numpy())
                parts.append(torch.sqrt(avar).permute(0, 2, 1).contiguous().cpu().numpy())
            else:
                # every channel a contiguous series: K4 then streams them with bulk copies
                gyro, accel = self._noise_block(r0, r1, engine.LAYOUT_CHANNEL_MAJOR)
                tau, a, g, *noise = algo.run_batch(self.fs[0], accel, gyro, channel_major=True)
                parts.append(np.concatenate([a, g], axis=2))
                if fit:
                    fits.append(np.concatenate(noise, axis=1))
        both = np.concatenate(parts) if parts else np.zeros((0, len(tau), 6))
        noise = (np.concatenate(fits) if fits else np.zeros((0, 6, 6))) if fit else None
        if dist.world() > 1:
            both, noise = _gather_allan(both, noise, self.sim_count)
        per_series = (noise[:, 0:3], noise[:, 3:6]) if fit else ()
        self._publish_allan(self.algo_name(i), algo, tau, both[:, :, 0:3], both[:, :, 3:6], *per_series)

    # ---- magnetometer calibration (K10) ---------------------------------------------------------
    def _publish_magcal(self, name, soft_iron, hard_iron):
        """soft_iron [R, 3, 3] and hard_iron [R, 4] under run keys, in the reference's shapes (3, 3) and (1, 4)."""
        self.data['soft_iron'] = _keyed(name, np.asarray(soft_iron).reshape(-1, 3, 3))
        self.data['hard_iron'] = _keyed(name, np.asarray(hard_iron).reshape(-1, 1, 4))

    def _run_magcal(self, i, algo):
        """All runs of this rank in one K10 launch that regenerates K8's samples (nothing is materialised):
        soft_iron and hard_iron of every run (gathered over ranks) and the ensemble statistics of the calibration
        errors; mag_cal is materialised per history block on request (K8, then the fed K10)."""
        if not getattr(self.imu, 'magnetometer', False):
            raise ValueError('MagCal calibrates the magnetometer: it needs IMU(axis=9)')
        check_segments(algo.segments, self._traj['ref_gyro'].shape[0])
        lo, hi = self._shard
        si, hard, stats = np.zeros((0, 9)), np.zeros((0, 4)), np.zeros((3, 13))
        if hi > lo:
            res = engine.mag_calibrate_mc(hi - lo, algo.segments, self._dev['ref_mag'], self.imu.mag_err, self.seed,
                                          run_offset=self.run_base + lo)
            stats = engine.error_stats(res.err).cpu().numpy()
            si, hard = res.soft_iron.reshape(-1, 9).cpu().numpy(), res.hard_iron.cpu().numpy()
        self._magcal[i] = dist.combine_local_stats(stats, hi - lo)
        if dist.world() > 1:
            both = dist.gather_rows(torch.from_numpy(np.ascontiguousarray(np.concatenate([si, hard], axis=1))),
                                    self.sim_count)
            si, hard = both[:, 0:9], both[:, 9:13]
        name = self.algo_name(i)
        self._publish_magcal(name, si, hard)
        self.data['mag_cal'] = LazyRuns(self, (i, 'mag_cal'), self.sim_count, prefix=name)

    # ---- loosely-coupled GNSS/INS filter (K7) -------------------------------------------------
    def _ekf_inputs(self):
        """Device copies of what K7 reads beside the IMU truth: GPS truth rows, their IMU sample
        indices, visibility."""
        t = self._traj
        if self.ref_frame != 0:
            raise ValueError('ins_loose works in ref_frame 0 (LLA positions, NED velocities)')
        if not (getattr(self.imu, 'gps', False) and 'ref_gps' in t and self.fs[1] > 0):
            raise ValueError('ins_loose needs IMU(gps=True), fs = [fs_imu, fs_gps, ...] and a trajectory '
                             'with ref_gps / gps_time / gps_visibility')
        d = self._dev
        return d['ref_gps'], d['gps_idx'], d['gps_vis']

    def _ekf_launch(self, algo, r0, runs, stats_start=0, dump_runs=0, dump_stride=1, proc_start=None,
                    proc_pos_frame=0, bias_err=False):
        gps = self._ekf_inputs()
        d = self._dev
        ini = algo.ini if algo.ini is not None else self._traj.get('ini')
        if algo.align_yaw is not None:
            t = self._traj
            algo.check_alignment(len(t['ref_gyro']), np.rint(np.asarray(t['gps_time']) * self.fs[0]),
                                 t['gps_visibility'], t['ref_gps'][:, 3:5])
        elif ini is None:
            raise ValueError('InsLoose needs ini_pos_vel_att (the trajectory carries no initial state)')
        vib_gyro, vib_acc = self._vib_pair(runs, r0)       # K5 (PSD) runs on the stream K7 runs on
        return engine.ins_loose(self.fs[0], runs, self.seed, self.imu.gyro_err, self.imu.accel_err,
                                self.imu.gps_err, ini, d['ref_gyro'], d['ref_accel'], d['ref_nav'],
                                *gps, run_offset=self.run_base + r0,
                                ini_att_std=algo.ini_att_std, earth_rot=algo.earth_rot,
                                stats_start=stats_start, dump_runs=dump_runs, dump_stride=dump_stride,
                                vel_rw=algo.vel_model_std, att_rw=algo.att_model_std,
                                vib_gyro=vib_gyro, vib_accel=vib_acc, proc_start=proc_start,
                                proc_pos_frame=proc_pos_frame, align=algo.align(), bias_err=bias_err)

    def _ekf_blocks(self, algo, **kw):
        """K7 over this rank's shard (kw: _ekf_launch's), in run blocks sized to the free device memory with PSD
        vibration, whose series K5 materialises (as for K9): the EkfResult of every block."""
        lo, hi = self._shard
        block = self._allan_block(48, 3) if self._uses_psd() else hi - lo
        parts = []
        for r0 in range(lo, hi, block):
            runs = min(hi, r0 + block) - r0
            parts.append(self._ekf_launch(algo, r0, runs, **kw))
            if block < hi - lo:     # the next block's series take the memory of this block's
                for sensor in (0, 1):
                    self._psd_cache.pop((sensor, runs, r0), None)
        return parts

    def _run_ins_loose(self, i, algo):
        """demo_ins_loose.py semantics, all runs of this rank in one K7 launch (in run blocks sized to the free
        device memory with PSD vibration, whose series K5 materialises, as for K9): end-point errors and their
        ensemble statistics (as for free integration), bias estimates, the consistency record and, when the IMU
        draws a turn-on bias, the bias-estimate errors."""
        name = self.algo_name(i)
        if algo.imu is not None and algo.imu is not self.imu:
            raise ValueError('a generating Sim filters with the IMU that makes its data: InsLoose(imu=...) must be '
                             "the Sim's imu or None")
        lo, hi = self._shard
        self._mc[i] = {'base': 0, 'end_err': None}
        err, stats, con, bias = np.zeros((0, 9)), np.zeros((3, 9)), np.zeros((0, 19)), np.zeros((0, 6))
        turn_on = any(_lib.set_run_errors(e) for e in (self.imu.gyro_err, self.imu.accel_err))   # only 'b_std' here
        bias_err = np.zeros((0, 6)) if turn_on else None
        if hi > lo:
            start = int(round(min(30.0, 0.1 * len(self.data['time']) / self.fs[0]) * self.fs[0]))
            parts = self._ekf_blocks(algo, stats_start=start, bias_err=turn_on)
            end_err = torch.cat([r.end_err for r in parts])
            stats = engine.error_stats(end_err).cpu().numpy()
            err = end_err.cpu().numpy()
            con = torch.cat([r.consist for r in parts]).cpu().numpy()
            bias = torch.cat([r.end_bias for r in parts]).cpu().numpy()
            if turn_on:
                bias_err = torch.cat([r.end_bias_err for r in parts]).cpu().numpy()
        self._mc[i].update({'end_err': err, 'consist': con, 'end_bias': bias, 'bias_err': bias_err})
        self.err_stats[name] = dist.combine_local_stats(stats, hi - lo)
        algo.run_times += self.sim_count
        for out in ('att_euler', 'pos', 'vel', 'wb', 'ab'):
            self.data[out] = LazyRuns(self, (i, out), self.sim_count, prefix=name)

    def ekf_consistency(self, algo_index=0):
        '''
        The filter's consistency record over this rank's runs (GPS epochs after the settling time,
        after the update): {'nees': [R,3] mean NEES of the position / velocity / attitude blocks
        (expected 3 each), 'inside3': [R,15] fraction of epochs with |error| <= 3 sigma per state
        (p, v, phi, bg, ba), 'epochs': count, 'end_bias': [R,6] bias estimates at the last sample,
        'bias_err': [R,6] those estimates minus each run's true gyro then accel bias (the IMU's 'b', the run's
        turn-on bias and the drift) when the IMU draws a turn-on bias ('b_std'), else None}.
        '''
        c = self._mc[algo_index]['consist']
        ep = np.maximum(c[:, 18:19], 1.0)
        return {'nees': c[:, 0:3] / ep, 'inside3': c[:, 3:18] / ep, 'epochs': int(c[0, 18]) if len(c) else 0,
                'end_bias': self._mc[algo_index]['end_bias'], 'bias_err': self._mc[algo_index]['bias_err']}

    # ---- lazy histories -------------------------------------------------------
    def _history(self, name, run):
        """(n,3) history of one run: from the histories() arrays if they hold it, else from the history block
        of neighbouring runs that one launch of name's source fills.  name: a sensor name, or
        (algo index, output name)."""
        if self._all_hist is not None:
            ai_w, lo_w, arrs = self._all_hist
            key_w = name[1] if isinstance(name, tuple) and name[0] == ai_w else name
            if isinstance(key_w, str) and key_w in arrs and 0 <= run - lo_w < arrs[key_w].shape[0]:
                return arrs[key_w][run - lo_w]
        blk, i = divmod(run, self.history_block)
        if (blk, name) not in self._blocks:
            r0 = blk * self.history_block
            filled = self._history_block(name, r0, min(self.sim_count, r0 + self.history_block) - r0)
            self._blocks.update({(blk, k): v for k, v in filled.items()})
        return self._blocks[(blk, name)][i]

    def _history_block(self, name, r0, runs):
        """One launch of what produces `name` for runs [r0, r0+runs): {name: [runs, ...] host array} of every
        history that launch makes.  A K12 block also holds the IMU samples of its runs (and the odometer's,
        for the odometer variant); odo histories come from the odometer plugin's K12 block."""
        if name == 'odo':      # pathgen.odo_gen stream: a zero-length odometer experiment
            ai = [i for i, a in enumerate(self.algo or []) if isinstance(a, FreeIntegrationOdo)]
            if not ai:
                raise KeyError('odo histories are produced with the free_integration_odo plugin')
            name = (ai[0], 'pos')
        if isinstance(name, tuple) and isinstance(self.algo[name[0]], MagCal):
            mag = engine.mag_noise(runs, self._dev['ref_mag'], self.imu.mag_err, self.seed,
                                   run_offset=self.run_base + r0)
            res = engine.mag_calibrate(self.algo[name[0]].segments, mag, want_cal=True)
            return {name: res.mag_cal.cpu().numpy()}
        if isinstance(name, tuple) and isinstance(self.algo[name[0]], InsLoose):
            res = self._ekf_launch(self.algo[name[0]], r0, runs, dump_runs=runs)
            return {(name[0], k): v.cpu().numpy() for k, v in (('att_euler', res.att), ('pos', res.pos),
                                                               ('vel', res.vel), ('wb', res.wb), ('ab', res.ab))}
        if isinstance(name, tuple) and self._fed(name[0]):
            out = {}
            for b0, att, pos, vel, gyro, accel in self._fed_blocks(name[0], r0, r0 + runs):
                for k, v in (((name[0], 'att_euler'), att), ((name[0], 'pos'), pos), ((name[0], 'vel'), vel),
                             ('gyro', gyro), ('accel', accel)):
                    out.setdefault(k, []).append(v.cpu().numpy())
            return {k: np.concatenate(v) for k, v in out.items()}
        if isinstance(name, tuple):
            res = self._mc_launch(name[0], r0, runs, dump_runs=runs, dump_nav=True, dump_imu=True)
            out = {(name[0], k): v.cpu().numpy() for k, v in (('att_euler', res.att), ('pos', res.pos),
                                                              ('vel', res.vel))}
            out.update({'gyro': res.gyro.cpu().numpy(), 'accel': res.accel.cpu().numpy()})
            if res.odo is not None:
                out['odo'] = res.odo.cpu().numpy()
            return out
        if name == 'gps':
            return {'gps': engine.gps_noise(runs, self._dev['ref_gps'], self.imu.gps_err, self.ref_frame,
                                            self.seed, run_offset=self.run_base + r0).cpu().numpy()}
        if name == 'mag':
            return {'mag': engine.mag_noise(runs, self._dev['ref_mag'], self.imu.mag_err, self.seed,
                                            run_offset=self.run_base + r0).cpu().numpy()}
        gyro, accel = self._noise_block(r0, r0 + runs)
        return {'gyro': gyro.cpu().numpy(), 'accel': accel.cpu().numpy()}

    def histories(self, algo_index=0, imu=False, stride=1, quat=False):
        '''
        Every run of this rank at once: {'att_euler', 'pos', 'vel'} -> [R_local, rows, 3] host arrays
        (plus 'gyro', 'accel' with imu=True, 'att_quat' [R_local, rows, 4] with quat=True) -- what
        the reference's Sim.run leaves in its data manager (ins_sim.py:184-187, att_quat associated
        :729-794), here by ONE launch with history output for all runs and one device-to-host copy
        per array into pinned memory.  stride > 1 keeps samples 0, stride, 2 stride, ... (rows =
        ceil(n / stride), 'time' decimated alike): error histories of many runs for plotting without
        72 bytes per run-step.  With stride 1 get_data() then serves single runs from these arrays.
        '''
        lo, hi = self._shard
        algo = self.algo[algo_index]
        if not isinstance(algo, FreeIntegration) or self._logged is not None:
            raise ValueError('histories() is for the fused free-integration experiment')
        runs = hi - lo
        if runs == 0:
            n = self._traj['ref_gyro'].shape[0]
            return {k: np.zeros((0, n, 3)) for k in ('att_euler', 'pos', 'vel')}
        stride = max(1, int(stride))
        if self._fed(algo_index):
            parts = {}
            for _, att, pos, vel, gyro, accel in self._fed_blocks(algo_index, lo, hi):
                names = [('att_euler', att), ('pos', pos), ('vel', vel)] + ([('gyro', gyro), ('accel', accel)]
                                                                             if imu else [])
                for k, t in names:
                    parts.setdefault(k, []).append(t[:, ::stride].cpu().numpy())
            out = {k: np.concatenate(v) for k, v in parts.items()}
            if quat:
                out['att_quat'] = np.stack([euler2quat_zyx(a) for a in out['att_euler']])
            if stride == 1:
                self._all_hist = (algo_index, lo, out)
            else:
                out['time'] = self.data['time'][::stride]
            return out
        pool = _hist_pool(self)      # device + pinned buffers: this Sim's, or a dead Sim's (never a live one's)
        res = self._mc_launch(algo_index, lo, runs, dump_runs=runs, dump_stride=stride, dump_nav=True,
                              dump_imu=imu, out=pool.get('res'), dump_quat=quat)
        pool['res'] = res
        pinned = pool.setdefault('pinned', {})
        names = [('att_euler', res.att), ('pos', res.pos), ('vel', res.vel)]
        if imu:
            names += [('gyro', res.gyro), ('accel', res.accel)]
        if quat:
            names += [('att_quat', res.quat)]
        for k, t in names:     # pinned staging is kept per process: pinning tens of MB costs milliseconds
            if k not in pinned or pinned[k].shape != t.shape:
                pinned[k] = torch.empty(t.shape, dtype=torch.float64, pin_memory=True)
        for k, t in names:
            pinned[k].copy_(t, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        out = {k: pinned[k].numpy() for k, _ in names}
        if stride == 1:
            self._all_hist = (algo_index, lo, out)
        else:
            out['time'] = self.data['time'][::stride]
        return out

    # ---- results --------------------------------------------------------------
    def get_names_of_available_data(self):
        return list(self.data.keys())

    def get_data(self, data_names):
        '''
        Get data by names (ins_sim.py:317-327): list of arrays / dicts of runs.
        '''
        return [self.data[n] if n in self.data else None for n in data_names]

    def save_data(self, data_dir, names=None, runs=None):
        """Write data to `<data_dir>/<name>[-<key>].csv` in the reference's file format
        (Sim_data.save_to_file, sim_data.py:117-165: output units, `legend (unit)` header), which
        both Sims read back as a logged-data directory.  names: data names (default: everything
        that has a file format); runs: keys of per-run data to write (default: all -- histories
        are materialised by re-running blocks of runs, mind the count)."""
        names = [n for n in self.data.keys() if n in logged.OUTPUT_FORMAT] if names is None else list(names)
        written = []
        for n in names:
            if n not in self.data or n not in logged.OUTPUT_FORMAT:
                raise KeyError('no file format for %r' % n)
            v = self.data[n]
            if isinstance(v, (dict, Mapping)):
                keys = list(v.keys()) if runs is None else [k for k in v.keys()
                                                          if k in runs or (isinstance(k, str) and
                                                                           k.rsplit('_', 1)[-1].isdigit() and
                                                                           int(k.rsplit('_', 1)[-1]) in runs)]
                v = {k: v[k] for k in keys}
            written += logged.write_data(data_dir, n, v, self.ref_frame)
        return written

    def end_point_errors(self, algo_index=0):
        '''
        [R_local, 9] end-point errors (att wrapped [rad], pos, vel) of this rank's runs
        (numpy) -- 72 bytes per run, the raw material of the ensemble statistics.
        '''
        return self._mc[algo_index]['end_err']

    def get_error_stats(self, data_name, err_stats_start=-1, angle=False, use_output_units=False,
                        extra_opt='', algo_index=0):
        '''
        InsDataMgr.get_error_stats (ins_data_manager.py:385-452) for att_euler / pos / vel of an algorithm and
        for the sensor data gyro / accel / mag / gps.
        err_stats_start == -1: end-point statistics over runs {'max','avg','std'} (3,) (sensor data: (3,) or
        (6,)).  Otherwise: per-run process statistics from that time [s]: dicts keyed by run key ('<algo>_<r>'
        for algorithm outputs, the run index for sensor data).  GPS process statistics start at the first
        GPS sample at or after that time.  For InsLoose(align_yaw=...) the statistics start at the later of that
        time and the fix sample (the first sample with a full state; earlier history rows are NaN).
        '''
        if data_name == 'odo':
            raise ValueError('odo has no error statistics: the odometer history is one column per run, and the '
                             "reference's own end-point statistics index it as a 2-D array "
                             '(ins_data_manager.py:737), so there is no defined result')
        if data_name in _MAGCAL_UNITS:
            return self._magcal_stats(data_name, err_stats_start, algo_index)
        if data_name in _SENSOR_UNITS:
            units, out_units = _SENSOR_UNITS[data_name]
            if data_name == 'gps' and self.ref_frame == 1:      # ins_data_manager.py:221-230
                units = out_units = ['m', 'm', 'm', 'm/s', 'm/s', 'm/s']
            st = self._sensor_stats(data_name, err_stats_start)
            return self._with_units(st, units, out_units, use_output_units)
        if data_name not in _UNITS:
            raise ValueError('error statistics exist for att_euler, pos, vel, gyro, accel, mag and gps')
        c0 = {'att_euler': 0, 'pos': 3, 'vel': 6}[data_name]
        desc, units, out_units = _UNITS[data_name]
        if data_name == 'pos' and self.ref_frame == 1:
            units, out_units = ['m'] * 3, ['m'] * 3
        name = self.algo_name(algo_index)
        # extra_opt 'ned' / 'ecef' in ref_frame 0: position error in metres (ignored in ref_frame 1, as in
        # the reference).  The reference keeps the first option's error array per data name
        # (ins_data_manager.py:427-431); here every call gets the option it asks for.
        frame = {'ned': engine.POS_FRAME_NED, 'ecef': engine.POS_FRAME_ECEF}.get(extra_opt, 0) \
            if self.ref_frame == 0 else 0
        if data_name == 'pos' and frame:
            units = out_units = ['m'] * 3
        if algo_index not in self._mc:
            # a reference-style plugin: its outputs are on the host
            errs, starts = zip(*(self._host_error(algo_index, r, data_name, frame) for r in range(self.sim_count)))
            if err_stats_start == -1:
                st = dict(zip(('max', 'avg', 'std'), _host_stats(np.stack([e[-1] for e in errs]))))
            else:
                ps = [_host_stats(e[_first_at(t, err_stats_start):]) for e, t in zip(errs, starts)]
                st = {s: _keyed(name, [p[k] for p in ps]) for k, s in enumerate(('max', 'avg', 'std'))}
        elif err_stats_start == -1:
            if frame:
                st = self._end_point_pos_stats(extra_opt, algo_index)
            else:
                s = self.err_stats[name]
                st = {'max': s[0, c0:c0 + 3].copy(), 'avg': s[1, c0:c0 + 3].copy(),
                      'std': s[2, c0:c0 + 3].copy()}
        else:
            st = self._process_stats(algo_index, err_stats_start, c0, frame)
        return self._with_units(st, units, out_units, use_output_units)

    def _magcal_stats(self, data_name, start_s, algo_index):
        """get_error_stats('soft_iron' | 'hard_iron', -1) of a MagCal on generated data: the statistics over runs
        of E = S si / k - I (9 values, row-major) or of (hard_iron[0:3] / k - hi, hard_iron[3] / k - |b|) [uT],
        with k = trace(S si) / 3 (b: the true field at the first sample)."""
        if algo_index not in getattr(self, '_magcal', {}):
            raise ValueError('%s error statistics need a MagCal run on generated data (algo_index %d is not one)'
                             % (data_name, algo_index))
        if start_s != -1:
            raise ValueError('%s error statistics are over runs only (err_stats_start=-1)' % data_name)
        st = self._magcal[algo_index]
        cols = slice(0, 9) if data_name == 'soft_iron' else slice(9, 13)
        return {'max': st[0, cols].copy(), 'avg': st[1, cols].copy(), 'std': st[2, cols].copy(),
                'units': str(_MAGCAL_UNITS[data_name])}

    @staticmethod
    def _with_units(st, units, out_units, use_output_units):
        """The statistics in output units on request (sim_data.convert_unit: rad -> deg), with the units string."""
        if use_output_units:
            scale = np.array([R2D if (u, o) in (('rad', 'deg'), ('rad/s', 'deg/s')) else 1.0
                              for u, o in zip(units, out_units)])
            for k in ('max', 'avg', 'std'):
                if isinstance(st[k], dict):
                    st[k] = {r: v * scale for r, v in st[k].items()}
                else:
                    st[k] = st[k] * scale
            st['units'] = str(out_units)
        else:
            st['units'] = str(units)
        return st

    def _host_error(self, ai, r, data_name, frame=0):
        """(e, t) of run r of a host-held output of algorithm ai (logged-data results, reference-style plugins):
        e = x - truth as calc_data_err / array_error make it (ins_data_manager.py:454-553) -- att_euler wrapped
        to [-pi, pi], pos in NED / ECEF metres for frame 1 / 2, the truth interpolated to the plugin's algo_time
        when the row counts differ (:497-506) -- and the times of its rows (algo_time if the plugin outputs it,
        :774-777)."""
        key = '%s_%d' % (self.algo_name(ai), r)
        x = np.asarray(self.data[data_name][key], dtype=np.float64)
        ref = self._traj[_REF_OF[data_name]]
        at = self.data.get('algo_time')
        t = np.asarray(at[key], dtype=np.float64) if isinstance(at, Mapping) and key in at else None
        if ref.shape[0] != x.shape[0]:
            if t is None:
                raise ValueError('%s of %s has %d rows and its truth %d: interpolating needs algo_time'
                                 % (data_name, key, x.shape[0], ref.shape[0]))
            ref = np.stack([np.interp(t, self.data['time'], ref[:, i]) for i in range(ref.shape[1])], axis=1)
        if data_name == 'att_euler':
            e = (x - ref + math.pi) % (2.0 * math.pi) - math.pi
        elif data_name == 'pos' and frame:
            e = lla_error_metres(x, ref, frame)
        else:
            e = x - ref
        return e, (self.data['time'] if t is None else t)

    # ---- sensor-data error statistics (K9 for gyro / accel, K8 / K6 + K3p for mag / gps) ------------
    def _sensor_stats(self, name, start_s):
        """get_error_stats of gyro / accel / mag / gps: end-point statistics over runs (start_s == -1) or
        per-run process statistics keyed by run index."""
        if name not in self.data:
            raise ValueError('%s is not available in this simulation' % name)
        if self._logged is not None:
            return self._logged_sensor_stats(name, start_s)
        src, cols = {'gyro': ('imu', slice(3, 6)), 'accel': ('imu', slice(0, 3)),
                     'mag': ('mag', slice(0, 3)), 'gps': ('gps', slice(0, 6))}[name]
        if start_s == -1:
            hit = next((v for k, v in self._sens.items() if k[0] == src), None)
            end_err, _ = hit if hit is not None else self._sensor_launch(src, -1)
            lo, hi = self._shard
            stats = np.zeros((3, cols.stop - cols.start))
            if hi > lo:
                stats = engine.error_stats(engine.to_device(end_err[:, cols])).cpu().numpy()
            stats = dist.combine_local_stats(stats, hi - lo)
            return {'max': stats[0], 'avg': stats[1], 'std': stats[2]}
        t = self._traj['gps_time'] if name == 'gps' else self.data['time']
        start = _first_at(t, start_s)
        if (src, start) not in self._sens:
            self._sensor_launch(src, start)
        ps = self._sens[(src, start)][1][:, :, cols]
        return {s: {r: ps[r, k].copy() for r in range(ps.shape[0])} for k, s in enumerate(('max', 'avg', 'std'))}

    def _sensor_launch(self, src, start):
        """This rank's runs of one source ('imu', 'mag', 'gps') reduced from row `start` (-1: end points only):
        caches and returns (end_err [R_local, C], process statistics [R, 3, C] of all ranks or None).  The IMU
        is one K9 launch (in run blocks only with PSD vibration, whose series K5 materialises); mag and gps
        are materialised by K8 / K6 in run blocks sized to the free device memory and reduced by K3p."""
        lo, hi = self._shard
        d = self._dev
        C = {'imu': 6, 'mag': 3, 'gps': 6}[src]
        if src == 'imu':
            block = self._allan_block(48, 3) if self._uses_psd() else max(hi - lo, 1)
        else:
            block = self._allan_block(8 * C, 3)
        ends, procs = [], []
        for r0 in range(lo, hi, block):
            runs = min(hi, r0 + block) - r0
            if src == 'imu':
                vib_gyro, vib_acc = self._vib_pair(runs, r0)
                e, p = engine.imu_err_stats(self.fs[0], runs, d['ref_gyro'], d['ref_accel'], self.imu.gyro_err,
                                            self.imu.accel_err, self.seed, run_offset=self.run_base + r0,
                                            vib_gyro=vib_gyro, vib_accel=vib_acc, stats_start=start)
            else:
                ref = d['ref_mag'] if src == 'mag' else d['ref_gps']
                if src == 'mag':
                    x = engine.mag_noise(runs, ref, self.imu.mag_err, self.seed, run_offset=self.run_base + r0)
                else:
                    x = engine.gps_noise(runs, ref, self.imu.gps_err, self.ref_frame, self.seed,
                                         run_offset=self.run_base + r0)
                e, p = engine.proc_stats(x, ref, max(start, 0))
                del x
            ends.append(e)
            procs.append(p)
        end_err = torch.cat(ends).cpu().numpy() if ends else np.zeros((0, C))
        proc = None
        if start >= 0:
            local = torch.cat(procs).reshape(hi - lo, 3 * C) if procs else None
            proc = dist.gather_rows(local, self.sim_count).reshape(-1, 3, C)
        self._sens[(src, start)] = (end_err, proc)
        return self._sens[(src, start)]

    def _logged_sensor_stats(self, name, start_s):
        """The statistics of a logged directory's <name>-<key>.csv sets against ref_<name>.csv, on the host."""
        ref = self._logged.get('ref_' + name)
        if ref is None:
            raise ValueError('the data directory holds no ref_%s.csv' % name)
        x = self._logged_sets(name)
        e = x - ref[None]
        if start_s == -1:
            return dict(zip(('max', 'avg', 'std'), _host_stats(e[:, -1])))
        t = self._logged.get('gps_time') if name == 'gps' else self.data['time']
        if t is None:
            raise ValueError('the data directory holds no gps_time.csv')
        ps = [_host_stats(er[_first_at(t, start_s):]) for er in e]
        return {s: {r: p[k] for r, p in enumerate(ps)} for k, s in enumerate(('max', 'avg', 'std'))}

    def _end_point_pos_stats(self, opt, algo_index):
        """'ned' / 'ecef' position error of LLA results, ins_data_manager.py:543-552."""
        err = self._mc[algo_index]['end_err']
        if dist.world() > 1:
            err = dist.gather_rows(torch.from_numpy(err), self.sim_count)
        r = self._traj['ref_pos'][-1]
        x = err[:, 3:6] + r            # end position = error + truth
        err = lla2ecef(x) - lla2ecef(r)[0]
        if opt == 'ned':
            err = err.dot(ecef_to_ned(r[0], r[1]).T)
        return {'max': np.max(np.abs(err), 0), 'avg': np.average(err, 0), 'std': np.std(err, 0)}

    def _process_stats(self, algo_index, start_s, c0, frame=0):
        """Per-run process statistics of columns c0:c0+3; frame: the position frame (engine.POS_FRAME_*).
        One launch holds all nine columns: the attitude and velocity columns of any frame's launch serve."""
        key = (algo_index, float(start_s), frame)
        if c0 != 3:
            key = next((k for k in ((algo_index, float(start_s), f) for f in (frame, 0, 1, 2))
                        if k in self._proc), key)
        if key not in self._proc:
            start = _first_at(self.data['time'], start_s)
            if self._logged is not None:
                start = max(start, self._mc.get(algo_index, {}).get('start', 0))     # aligned: from the fix
                # the histories are on the host already (array_error + __array_stats,
                # ins_data_manager.py:512-541, :797-808)
                ps = np.zeros((self.sim_count, 3, 9))
                for r in range(self.sim_count):
                    e = np.concatenate([self._host_error(algo_index, r, dn, frame)[0]
                                        for dn in ('att_euler', 'pos', 'vel')], axis=1)[start:]
                    ps[r] = _host_stats(e)
            else:
                lo, hi = self._shard
                ps = None
                algo = self.algo[algo_index]
                if hi > lo and isinstance(algo, InsLoose):
                    # reduced inside the filter kernel (which starts aligned runs at the fix sample): the
                    # histories of all runs would not fit
                    ps = torch.cat([r.proc_stats for r in self._ekf_blocks(algo, proc_start=start,
                                                                           proc_pos_frame=frame)])
                    ps = ps.reshape(hi - lo, 27)
                elif hi > lo and self._fed(algo_index):
                    # K2's histories of each block, reduced on the host as for logged results
                    ps = torch.from_numpy(np.concatenate([
                        np.stack([_host_stats(e) for e in self._fed_errors(a, p, v, frame, slice(start, None))])
                        for _, a, p, v, _, _ in self._fed_blocks(algo_index, lo, hi)]).reshape(hi - lo, 27))
                elif hi > lo:
                    ps = self._mc_launch(algo_index, lo, hi - lo, stats_start=start,
                                         proc_pos_frame=frame).proc_stats.reshape(hi - lo, 27)
                ps = dist.gather_rows(ps, self.sim_count).reshape(-1, 3, 9)
            self._proc[key] = ps
        ps = self._proc[key]
        name = self.algo_name(algo_index)
        return {s: _keyed(name, ps[:, k, c0:c0 + 3].copy()) for k, s in enumerate(('max', 'avg', 'std'))}

    def results(self, data_dir=None, err_stats_start=0, gen_kml=False, extra_opt=''):
        '''
        Simulation summary (ins_sim.py:194-251, :339-413): the configuration and the error
        statistics of att_euler / pos / vel in output units.  Returns the available data
        names.  data_dir saves summary.txt; per-run data go to .csv files on request
        (save_data: a Monte-Carlo experiment has thousands of runs); .kml export is out of scope.
        '''
        if not self.sim_complete:
            print("Sim.run() has not been called yet: nothing to summarise.")
            return None
        if gen_kml:
            raise NotImplementedError('kml export is the reference\'s kml_gen (out of scope)')
        s = '\n------------------------------------------------------------\n'
        s += 'Sample frequency of IMU: [fs] = %s Hz\n' % str(self.fs[0])
        s += 'Reference frame: %s\n' % str(self.ref_frame)
        s += 'Simulation time duration: %s s\n' % str(len(self.data['time']) / self.fs[0])
        s += 'Simulation runs: %s\n' % str(self.sim_count)
        names = []
        if self._mc and self.err_stats:      # logged data may lack references
            ai, names = sorted(self._mc.keys())[0], ['att_euler', 'pos', 'vel']
        else:   # reference-style plugins only: the first one that outputs att_euler / pos / vel with a truth
            for i, a in enumerate(self.algo or []):
                got = [dn for dn in _REF_OF if dn in a.output and _REF_OF[dn] in (self._traj or {})]
                if i not in self._mc and got:
                    ai, names = i, got
                    break
        if names:
            s += '\n------------------------------------------------------------\n'
            s += 'The following are error statistics.'
            for dn in names:
                st = self.get_error_stats(dn, err_stats_start=err_stats_start,
                                          angle=(dn == 'att_euler'), use_output_units=True,
                                          extra_opt=extra_opt, algo_index=ai)
                s += '\n-----------statistics for %s (in units of %s)\n' % (_UNITS[dn][0], st['units'])
                if isinstance(st['max'], dict):
                    for run in sorted(st['max'].keys()):
                        s += '\tSimulation run %s:\n' % str(run)
                        s += '\t\t--Max error: %s\n' % str(st['max'][run])
                        s += '\t\t--Avg error: %s\n' % str(st['avg'][run])
                        s += '\t\t--Std of error: %s\n' % str(st['std'][run])
                else:
                    s += '\t--Max error: %s\n' % str(st['max'])
                    s += '\t--Avg error: %s\n' % str(st['avg'])
                    s += '\t--Std of error: %s\n' % str(st['std'])
        for i in sorted(getattr(self, '_magcal', {})):
            s += '\n------------------------------------------------------------\n'
            s += 'Calibration errors of %s over runs (S si / k - I; hard iron / k - hi, radius / k - |b|).' \
                % self.algo_name(i)
            for dn in ('soft_iron', 'hard_iron'):
                st = self.get_error_stats(dn, algo_index=i)
                s += '\n-----------statistics for %s (in units of %s)\n' % (dn, st['units'])
                s += '\t--Max error: %s\n' % str(st['max'])
                s += '\t--Avg error: %s\n' % str(st['avg'])
                s += '\t--Std of error: %s\n' % str(st['std'])
        self.sum += s
        if dist.rank() == 0:
            print(self.sum)
            if data_dir is not None:
                os.makedirs(data_dir, exist_ok=True)
                with open(os.path.join(data_dir, 'summary.txt'), 'w') as f:
                    f.write(self.sum + '\n')
        self.sim_results = True
        return self.get_names_of_available_data()

    def plot(self, what_to_plot, sim_idx=None, opt=None, extra_opt=''):
        raise NotImplementedError('plotting is the reference\'s sim_data_plot (matplotlib), out '
                                  'of scope: use get_data() and plot the arrays')


# History staging (device buffers + pinned host tensors: tens of MB, milliseconds to pin) is handed from
# a Sim that no longer exists to the next one that asks; a live Sim keeps its own, so the arrays
# histories() returned stay valid as long as their Sim does.
_HIST_POOLS = []      # [weakref to the owning Sim or None, dict]


def _hist_pool(sim):
    for entry in _HIST_POOLS:
        if entry[0] is not None and entry[0]() is sim:
            return entry[1]
    for entry in _HIST_POOLS:
        if entry[0] is None or entry[0]() is None:
            entry[0] = weakref.ref(sim)
            return entry[1]
    _HIST_POOLS.append([weakref.ref(sim), {}])
    return _HIST_POOLS[-1][1]


class _Merged(Mapping):
    """Several algorithms writing the same output name: one dict view over all of them."""

    def __init__(self, parts):
        self._parts = list(parts)

    def add(self, p):
        self._parts.append(p)

    def __iter__(self):
        for p in self._parts:
            yield from p

    def __len__(self):
        return sum(len(p) for p in self._parts)

    def __getitem__(self, key):
        for p in self._parts:
            if key in p:
                return p[key]
        raise KeyError(key)
