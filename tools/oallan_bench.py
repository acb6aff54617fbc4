"""The Allan experiment of BASELINE config 4 with the overlapping estimators (K4o: Allan and Hadamard forms)
beside the reference's (K4).

    python tools/oallan_bench.py [--runs 256] [--windows 3] [--out DIR]

Config 4: static 10 h @400 Hz (n = 14.4 M samples), 'low-accuracy' IMU, Sim.run(runs) with Allan(overlapping=True),
with Hadamard() and with Allan(), in alternated windows (overlapping, Hadamard, default, overlapping, ...) in one
process, so that drift of the shared card's clocks falls on all alike.  Allan() takes K1 fused into K4; the other
two materialise K1's series in run blocks and run K4o on them.  Per window: the wall time of Sim.run and, for the
K4o experiments, the summed CUDA-event time of their K4o calls (engine.oallan / engine.ohadamard, all five passes).
K4o's bytes are counted from shapes: the passes that must reach HBM read the series twice and write and read the
prefix once (8 + 8 + 16 + 16 B per series-sample), and every decade reads the prefix again at its lags (14 for
Allan, 18 for Hadamard: 16 B x (lags + 1) per series-sample and decade, served from L1 / L2 as far as the lag
windows are recent).  Prints the card's name and power limit (read in the same process) and one JSON line per
estimator with medians."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import engine, imu_model  # noqa: E402
from gnss_ins_sim_b200.sim import Sim  # noqa: E402
from gnss_ins_sim_b200.allan_analysis import Allan, Hadamard  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


class OallanTimer(object):
    """Wraps engine.oallan or engine.ohadamard: CUDA events around every call on the current stream, summed
    after a sync."""

    def __init__(self, inner):
        self.inner = inner
        self.events = []
        self.series_samples = 0

    def __call__(self, fs, x, n, nseries, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = self.inner(fs, x, n, nseries, *a, **k)
        e1.record()
        self.events.append((e0, e1))
        self.series_samples += n * nseries
        return out

    def take(self):
        torch.cuda.synchronize()
        ms = sum(a.elapsed_time(b) for a, b in self.events)
        ss = self.series_samples
        self.events, self.series_samples = [], 0
        return ms * 1e-3, ss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=256)
    ap.add_argument('--windows', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    lines = [{'card': card()}]
    print(json.dumps(lines[0]), flush=True)
    n, fs, seed = 14400000, 400.0, 5
    traj = {'ref_pos': np.zeros((n, 3)), 'ref_vel': np.zeros((n, 3)), 'ref_att': np.zeros((n, 3)),
            'ref_accel': np.tile(np.array([4.9, 0.0, -8.487]), (n, 1)), 'ref_gyro': np.zeros((n, 3))}
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    timers = {'overlapping': OallanTimer(engine.oallan), 'hadamard': OallanTimer(engine.ohadamard)}
    engine.oallan, engine.ohadamard = timers['overlapping'], timers['hadamard']
    ndec = len({len(str(m)) for m in engine.allan_num_tau(n, fs)})
    arms = (('overlapping', lambda: Allan(overlapping=True), 'ad_gyro'), ('hadamard', Hadamard, 'hd_gyro'),
            ('default', Allan, 'ad_gyro'))
    wall = {a: [] for a, _, _ in arms}
    k4o = {a: [] for a in timers}
    results = {}
    for w in range(args.windows + 1):          # window 0 warms up every arm (compiles nothing; allocates)
        for arm, make, out in arms:
            sim = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=make(), seed=seed)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sim.run(args.runs)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if arm in timers:
                kt, _ = timers[arm].take()
            if w > 0:
                wall[arm].append(dt)
                if arm in timers:
                    k4o[arm].append(kt)
            results[arm] = sim.get_data([out])[0]['algo0_0']
            del sim
    ss = args.runs * 6 * n
    for arm, lags, what in (('overlapping', 14, 'overlapping Allan (K1 materialised + K4o)'),
                            ('hadamard', 18, 'overlapping Hadamard (K1 materialised + K4o, Hadamard form)')):
        t = float(np.median(k4o[arm]))
        hbm = (8 + 8 + 16 + 16) * ss          # what must reach HBM at least once per call (see the docstring)
        lag = 16 * (lags + 1) * ndec * ss     # the lag reads of pass 4, L1 / L2 / HBM
        rec = {'estimator': what, 'runs': args.runs, 'samples': n, 'series_samples': ss, 'decades': ndec,
               'windows_s': wall[arm], 'median_s': float(np.median(wall[arm])),
               'k4o_windows_s': k4o[arm], 'k4o_median_s': t, 'k4o_series_samples_per_s': ss / t,
               'k4o_min_hbm_bytes': hbm, 'k4o_min_hbm_share_of_3.35TBps': hbm / t / HBM_BYTES_PER_S,
               'k4o_lag_read_bytes': lag, 'k4o_lag_read_TBps': lag / t / 1e12}
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    rec = {'estimator': 'default (K1 fused into K4)', 'runs': args.runs, 'samples': n,
           'windows_s': wall['default'], 'median_s': float(np.median(wall['default']))}
    lines.append(rec)
    print(json.dumps(rec), flush=True)
    # the curves of run 0, gyro x, side by side (deviations, rad/s): they agree where both are well determined
    a, h, b = results['overlapping'][:, 0], results['hadamard'][:, 0], results['default'][:, 0]
    rec = {'run0_gyro_x_ratio_overlapping_to_default': (a / b).tolist(),
           'run0_gyro_x_ratio_hadamard_to_overlapping': (h / a).tolist()}
    lines.append(rec)
    print(json.dumps(rec), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'oallan_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
