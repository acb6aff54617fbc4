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

It is driven by gnss_ins_sim_b200.sim.Sim (ref_frame 0, IMU(gps=True), fs = [fs_imu, fs_gps, 0]); the
per-run .run(set_of_input) of the reference protocol would need the measurements on the host and a
CPU filter, which this package does not have (no CPU fallback): it raises.
"""
import numpy as np


class InsLoose(object):
    '''
    Loosely coupled INS algorithm (device-backed, Monte-Carlo form).
    '''

    def __init__(self, ini_pos_vel_att=None, ini_att_std=(0.02, 0.005, 0.005), earth_rot=True,
                 vel_model_std=0.02, att_model_std=0.0):
        '''
        Args:
            ini_pos_vel_att: (9,) true initial LLA [rad, rad, m], body velocity, ZYX Euler angles; None:
                the initial state of the motion definition the Sim was given.  Every run starts from
                this state plus a draw from the initial covariance.
            ini_att_std: 1-sigma of the initial misalignment about N, E, D [rad].
            earth_rot: consider the Earth rotation in the mechanization.
            vel_model_std, att_model_std: extra velocity [m/s/sqrt(s)] and misalignment [rad/sqrt(s)]
                random walks of the filter model.  The reference's truth generator and its first-order
                mechanization disagree slightly (noise-free free integration of motion_def-ins.csv ends
                0.37 m/s off); 0.02 m/s/sqrt(s) covers that and keeps the filter consistent.

        Vibration: the measurements carry the Sim's env vibration (random, sinusoidal or PSD), as
        get_data(['accel']) / get_data(['gyro']) do, but the filter model does not know about it.  Tell
        it through these two random walks.  For white (random) vibration of 1-sigma sa [m/s^2] on the
        accelerometer and sg [rad/s] on the gyro, sampled at dt = 1 / fs:
            vel_model_std = sqrt(0.02**2 + sa**2 * dt),   att_model_std = sg * sqrt(dt)
        (plus any att_model_std of its own, in quadrature).  With the default model the velocity and
        attitude blocks become overconfident (DESIGN.md section 11 has the figures).
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

    def run(self, set_of_input):
        raise NotImplementedError(
            'InsLoose runs as one fused Monte-Carlo kernel through gnss_ins_sim_b200.sim.Sim (measurement '
            'generation + filter on the device); there is no per-run host filter (no CPU fallback)')

    def get_results(self):
        return [self.results]

    def reset(self):
        pass
