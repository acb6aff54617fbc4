"""Two small reference-style algorithm plugins (the InsAlgoMgr protocol: input, output, run, get_results,
reset) whose att_euler / pos / vel error statistics are frozen in tests/golden/sensor_stats_90deg.npz.
They need nothing but NumPy, so tests import them on machines without the reference.  Test infrastructure
only.

Both perturb the truth they are given by a deterministic function of the run's gyro and accel, so every run
has different errors:
  * FullRate outputs att_euler, pos and vel at the IMU rate;
  * HalfRate outputs algo_time and the same quantities at every second IMU sample, so the truth has to
    be interpolated to algo_time (ins_data_manager.py:497-506) and the start index of process statistics
    comes from algo_time (:774-775).
"""
import numpy as np

_INPUT = ['fs', 'time', 'gyro', 'accel', 'ref_pos', 'ref_vel', 'ref_att_euler']
_POS_SCALE = np.array([1.0e-7, 1.0e-7, 1.0])     # rad, rad, m per (m/s) of integrated accel error


def _outputs(set_of_input, step):
    fs, t, gyro, accel, ref_pos, ref_vel, ref_att = set_of_input
    dt = 1.0 / fs
    dw = np.cumsum(gyro, axis=0) * dt                     # integrated rate [rad]
    dv = np.cumsum(accel - accel[0], axis=0) * dt         # integrated specific-force change [m/s]
    att = ref_att + 0.01 * dw + np.array([3.0, -0.5, 0.25]) * np.sin(dw)     # wraps past +-pi on the turn
    pos = ref_pos + _POS_SCALE * dv
    vel = ref_vel + 0.1 * dv + 0.02 * gyro
    return t[::step], att[::step], pos[::step], vel[::step]


class FullRate(object):
    def __init__(self):
        self.input = list(_INPUT)
        self.output = ['att_euler', 'pos', 'vel']
        self.results = None

    def run(self, set_of_input):
        self.results = list(_outputs(set_of_input, 1)[1:])

    def get_results(self):
        return self.results

    def reset(self):
        self.results = None


class HalfRate(FullRate):
    def __init__(self):
        super().__init__()
        self.output = ['algo_time', 'att_euler', 'pos', 'vel']

    def run(self, set_of_input):
        self.results = list(_outputs(set_of_input, 2))
