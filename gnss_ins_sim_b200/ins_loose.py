"""InsLoose plugin -- the loosely-coupled GNSS/INS filter of demo_ins_loose.py, with the attribute
names of demo_algorithms/ins_loose.py:24-38 (.input / .output / .batch, .run / .get_results / .reset).

In the reference this algorithm is a stub: InsLoose.prediction() and .correction() are `pass`
(ins_loose.py:124-134) and demo_ins_loose.py prints "Still under development".  What runs here is a
15-state closed-loop error-state EKF specified from first principles (DESIGN.md section 11: position /
velocity / misalignment / gyro-bias / accel-bias errors, GPS position + velocity updates at the GPS
rate), as ONE CUDA kernel for all Monte-Carlo runs (csrc/ekf_kernel.cuh): each run generates its own
IMU and GPS measurements from the shared true trajectory (the reference's sensor models on Philox
streams), filters them, and leaves end-point errors, bias estimates and a consistency record (NEES,
3-sigma containment).  Parity with the reference is unpinnable; the filter is validated statistically.

It is driven by gnss_ins_sim_b200.sim.Sim (ref_frame 0, IMU(gps=True), fs = [fs_imu, fs_gps, 0]).  The same
filter also runs on SUPPLIED measurements (a drive log, another simulator, a saved experiment): run_batch() for
R runs in one launch, the reference's per-run .run(set_of_input), and Sim on a logged-data directory.  There it
needs its noise model, InsLoose(imu=IMU(..., gps=True)), and an initial state -- or InsLoose(align_yaw=...), with
which it initialises itself from its measurements as the reference's InsLoose.ins_loose does (ins_loose.py:54-126).
"""
import numpy as np
import torch

from . import engine


class ModelMissing(ValueError, NotImplementedError):
    """The filter has no noise model (InsLoose(imu=...)) for measurements it did not generate."""


def gps_sample_index(fs, time, gps_time):
    """IMU sample of every GPS row: the sample nearest to gps_time[j] by time, ties to the earlier one
    (rint(gps_time * fs) for the simulator's own data).  Raises ValueError for a row outside the series, a row
    more than half a sample (0.5 / fs) from every IMU sample (a gap in time), and rows that do not land on
    strictly increasing samples: the filter applies at most one GPS row per sample, in order."""
    time = np.asarray(time, dtype=np.float64).reshape(-1)
    gt = np.asarray(gps_time, dtype=np.float64).reshape(-1)
    n = time.size
    if n < 2 or not np.all(np.diff(time) > 0.0):
        raise ValueError('time must hold at least two strictly increasing IMU sample times')
    half = 0.5 / float(fs)
    tol = 1e-9 * half           # times read back from text files may be an ulp off the grid
    for j, t in enumerate(gt):
        if not (time[0] - half - tol <= t <= time[-1] + half + tol):
            raise ValueError('gps_time[%d] = %r s lies outside the IMU series [%r, %r] s' % (j, t, time[0], time[-1]))
    k = np.clip(np.searchsorted(time, gt, side='left'), 1, n - 1)
    idx = np.where(gt - time[k - 1] <= time[k] - gt, k - 1, k)
    for j in np.nonzero(np.abs(gt - time[idx]) > half + tol)[0]:
        raise ValueError('gps_time[%d] = %r s lies more than half a sample from every IMU sample' % (j, gt[j]))
    for j in np.nonzero(np.diff(idx) <= 0)[0]:
        raise ValueError('gps rows %d and %d (%r s, %r s) land on IMU samples %d and %d: every row needs a later '
                         'sample than the row before' % (j, j + 1, gt[j], gt[j + 1], idx[j], idx[j + 1]))
    return idx.astype(np.int64)


class InsLoose(object):
    '''
    Loosely coupled INS algorithm (device-backed, Monte-Carlo form).
    '''

    def __init__(self, ini_pos_vel_att=None, ini_att_std=(0.02, 0.005, 0.005), earth_rot=True,
                 vel_model_std=0.02, att_model_std=0.0, imu=None, align_yaw=None):
        '''
        Args:
            ini_pos_vel_att: (9,) true initial LLA [rad, rad, m], body velocity, ZYX Euler angles; None:
                the initial state of the motion definition the Sim was given (on a logged-data directory: its
                first reference row).  Every run of a Sim starts from this state plus a draw from the initial
                covariance; run_batch() / run() need it given here.
            ini_att_std: 1-sigma of the initial misalignment about N, E, D [rad].
            earth_rot: consider the Earth rotation in the mechanization.
            vel_model_std, att_model_std: extra velocity [m/s/sqrt(s)] and misalignment [rad/sqrt(s)]
                random walks of the filter model.  The reference's truth generator and its first-order
                mechanization disagree slightly (noise-free free integration of motion_def-ins.csv ends
                0.37 m/s off); 0.02 m/s/sqrt(s) covers that and keeps the filter consistent.
            imu: the filter's noise model on supplied measurements, an imu_model.IMU with gps=True (its gyro,
                accelerometer and GPS errors set Q, R and P0).  Needed by run_batch() / run(); a Sim on a
                logged-data directory falls back to its own imu.  A generating Sim filters with the IMU that
                makes its data: any other model there is an error.

        Vibration: the measurements carry the Sim's env vibration (random, sinusoidal or PSD), as
        get_data(['accel']) / get_data(['gyro']) do, but the filter model does not know about it.  Tell
        it through these two random walks.  For white (random) vibration of 1-sigma sa [m/s^2] on the
        accelerometer and sg [rad/s] on the gyro, sampled at dt = 1 / fs:
            vel_model_std = sqrt(0.02**2 + sa**2 * dt),   att_model_std = sg * sqrt(dt)
        (plus any att_model_std of its own, in quadrature).  With the default model the velocity and
        attitude blocks become overconfident (DESIGN.md section 11 has the figures).

        Turn-on bias: an IMU with gyro_b_std / accel_b_std (imu_model 'b_std') gives every run of a Sim its own
        constant bias, drawn as K1 draws it (Sim.imu_run_errors() lists them).  The filter's model knows its
        spread: the bias states start at b_drift^2 + b^2 + b_std^2 (and the aligned level and gap terms grow
        with it), so the gyro- and accel-bias states estimate each run's bias.  Sim.ekf_consistency()['bias_err']
        gives how far each run's estimate ends from the truth.  The bias states are Gauss-Markov: on runs much
        longer than the bias correlation time the filter lets the constant part decay and becomes overconfident
        on the bias and attitude states (DESIGN.md section 11, "Turn-on bias", has the config-5 figures).  On
        supplied measurements the model's b_std enters the same P0.  The other run-to-run and IEEE Std 952 errors (scale factor, misalignment, quantisation,
        rate random walk, rate ramp) are not among the 15 states: a Sim refuses such an IMU.

        align_yaw: None (default): every run starts at the initial state above plus a draw from the initial
            covariance.  A heading [rad] or 'gps': every run initialises itself from its own measurements, with no
            initial state (DESIGN.md section 11, "Alignment"):
              - roll and pitch from the mean of the first 10 accelerometer samples, at sample 9
                (ins_loose.py:76-91); yaw is align_yaw (1-sigma ini_att_std[2]) or, with 'gps', the course over
                ground atan2(v_E, v_N) of the fix row's GPS velocity (a land vehicle moving forward);
              - the fix row is the latest visible GPS row at or before sample 9, else the first visible one
                after it: position and velocity as measured there, the attitude propagated alone until then;
              - P0 from the sensor models (level: accelerometer bias and noise; yaw: ini_att_std[2] or the
                course variance from the GPS velocity noise; the gyro's growth over the gap).
            History rows before the state exists are NaN; the consistency record and the process statistics
            start at the fix sample.  The error model is small-angle: the heading converges only from yaw errors
            the yaw P0 covers, so use 'gps' for a start in motion (a 'gps' fix needs >= 1 m/s horizontal
            speed).  Not together with ini_pos_vel_att.
        '''
        self.input = ['fs', 'gyro', 'accel', 'time', 'gps_time', 'gps']   # ins_loose.py:31
        self.output = ['pos', 'vel', 'att_euler', 'wb', 'ab']             # ins_loose.py:32
        self.batch = True
        self.results = None
        self.ini = None if ini_pos_vel_att is None else np.asarray(ini_pos_vel_att, dtype=np.float64).reshape(-1)[:9]
        self.ini_att_std = tuple(float(v) for v in ini_att_std)
        self.earth_rot = bool(earth_rot)
        self.vel_model_std, self.att_model_std = float(vel_model_std), float(att_model_std)
        self.run_times = 0
        if imu is not None and not getattr(imu, 'gps', False):
            raise ValueError('InsLoose(imu=...) needs an IMU with gps=True: its GPS errors are the filter\'s R')
        self.imu = imu
        if align_yaw is not None:
            if ini_pos_vel_att is not None:
                raise ValueError('InsLoose: align_yaw and ini_pos_vel_att exclude each other')
            if not (align_yaw == 'gps' or (not isinstance(align_yaw, str) and np.isfinite(float(align_yaw)))):
                raise ValueError("align_yaw must be a heading in rad or 'gps'")
        self.align_yaw = align_yaw if align_yaw is None or align_yaw == 'gps' else float(align_yaw)

    def align(self):
        """engine's align argument: None, or (align_yaw, its variance ini_att_std[2]^2)."""
        return None if self.align_yaw is None else (self.align_yaw, self.ini_att_std[2] ** 2)

    def check_alignment(self, n, gps_idx, gps_vis, gps_vel):
        """The host checks of an aligned launch, ValueError before any launch: n >= 10 IMU samples, a visible GPS
        row and, with 'gps', a horizontal speed >= 1 m/s at the fix row in every run.  gps_vel [..., m, 2]
        (v_N, v_E; numpy or a CUDA tensor, of which only the fix row is copied).  Returns the fix sample."""
        if n < engine.ALIGN_N:
            raise ValueError('InsLoose(align_yaw=...) needs at least %d IMU samples (got %d)' % (engine.ALIGN_N, n))
        j, start = engine.align_fix(gps_idx, gps_vis)
        if j is None:
            raise ValueError('InsLoose(align_yaw=...) needs a visible GPS row')
        if self.align_yaw == 'gps':
            v = gps_vel[..., j, :]
            v = np.asarray(v.cpu().numpy() if torch.is_tensor(v) else v, dtype=np.float64)
            if not np.all(np.hypot(v[..., 0], v[..., 1]) >= 1.0):
                raise ValueError("InsLoose(align_yaw='gps') needs a horizontal speed of at least 1 m/s at the fix "
                                 "row (GPS row %d)" % j)
        return start

    def run(self, set_of_input):
        '''
        One run of the reference protocol: set_of_input = [fs, gyro (n,3) rad/s, accel (n,3) m/s^2, time (n,)
        s, gps_time (m,) s, gps (m,6) LLA rad, m, NED m/s].  Every GPS row is used; the run starts at ini, or
        aligns itself with align_yaw.
        '''
        fs, gyro, accel, time, gps_time, gps = set_of_input
        out = self.run_batch(fs, np.asarray(gyro, dtype=np.float64)[None], np.asarray(accel, dtype=np.float64)[None],
                             time, gps_time, np.asarray(gps, dtype=np.float64)[None])
        self.results = [o[0] for o in out]

    def get_results(self):
        '''
        [pos, vel, att_euler, wb, ab] of the last run(), in self.output order.
        '''
        return self.results

    def reset(self):
        pass

    def run_batch(self, fs, gyro, accel, time, gps_time, gps, gps_visibility=None, seed=None, to_host=True):
        '''
        R runs of supplied measurements in one launch.  gyro, accel [R, n, 3] (rad/s, m/s^2); time [n] s;
        gps_time [m] s; gps [R, m, 6] (LLA rad, m; NED m/s); gps_visibility [m] (None: every row is used).  GPS
        row j is applied at the IMU sample nearest to gps_time[j] (gps_sample_index).  seed None: every run
        starts at ini; an integer: ini plus the initial-covariance draw of run run_times + r under that seed,
        as a generated experiment draws it.  With align_yaw every run aligns itself (seed is unused).  Returns pos, vel, att_euler, wb, ab [R, n, 3] (numpy, or CUDA
        tensors if not to_host).
        '''
        imu = self.model()
        g, a, gp = engine.to_device(gyro), engine.to_device(accel), engine.to_device(gps)
        if g.dim() != 3 or g.shape[2] != 3 or a.shape != g.shape:
            raise ValueError('gyro and accel must both be [R, n, 3]')
        if gp.dim() != 3 or gp.shape[0] != g.shape[0] or gp.shape[2] != 6:
            raise ValueError('gps must be [R, m, 6] with the R of gyro / accel')
        if np.asarray(time).reshape(-1).size != g.shape[1]:
            raise ValueError('time needs one entry per IMU sample (%d)' % g.shape[1])
        if np.asarray(gps_time).reshape(-1).size != gp.shape[1]:
            raise ValueError('gps_time needs one entry per GPS row (%d)' % gp.shape[1])
        vis = np.ones(gp.shape[1]) if gps_visibility is None else np.asarray(gps_visibility, dtype=np.float64).reshape(-1)
        if vis.size != gp.shape[1]:
            raise ValueError('gps_visibility needs one entry per GPS row (%d)' % gp.shape[1])
        res = self.launch(fs, g, a, gp, gps_sample_index(fs, time, gps_time), vis, imu, self.ini,
                          0 if seed is None else seed, seed is not None, self.run_times)
        self.run_times += g.shape[0]
        out = (res.pos, res.vel, res.att, res.wb, res.ab)
        return tuple(o.cpu().numpy() for o in out) if to_host else out

    def model(self, fallback=None):
        """The filter's noise model: imu, else fallback; ModelMissing if neither."""
        imu = self.imu if self.imu is not None else fallback
        if imu is None:
            raise ModelMissing('InsLoose on supplied measurements needs its noise model: InsLoose(imu=IMU(..., '
                               'gps=True)).  (Inside gnss_ins_sim_b200.sim.Sim the filter generates its own data.)')
        if not getattr(imu, 'gps', False):
            raise ValueError('the filter model must be an IMU with gps=True')
        return imu

    def launch(self, fs, gyro, accel, gps, gps_idx, gps_vis, imu, ini, seed, ini_draw, run_offset, ref_nav=None):
        """engine.ins_loose_fed with this filter's options and histories of every run: gyro, accel [R,n,3], gps
        [R,m,6], ref_nav [n,9] (optional) CUDA; gps_idx, gps_vis [m] host arrays.  With align_yaw, ini is unused
        and the alignment's host checks run first."""
        if self.align_yaw is not None:
            self.check_alignment(gyro.shape[1], gps_idx, gps_vis, gps[:, :, 3:5])
        elif ini is None:
            raise ValueError('InsLoose on supplied measurements needs ini_pos_vel_att (or align_yaw)')
        R = gyro.shape[0]
        return engine.ins_loose_fed(fs, gyro, accel, gps, torch.from_numpy(np.asarray(gps_idx, dtype=np.int64)).cuda(),
                                    engine.to_device(gps_vis), imu.gyro_err, imu.accel_err, imu.gps_err, ini,
                                    seed=seed, ini_draw=ini_draw, run_offset=run_offset,
                                    ini_att_std=self.ini_att_std, earth_rot=self.earth_rot, ref_nav=ref_nav,
                                    dump_runs=R, vel_rw=self.vel_model_std, att_rw=self.att_model_std,
                                    align=self.align())
