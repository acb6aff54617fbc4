"""Allan noise identification (K13) on BASELINE config 4 through Sim, and K13 alone.

    python tools/allan_fit_bench.py [--runs 256] [--windows 3] [--out DIR]

Config 4: static 10 h @400 Hz (n = 14.4 M samples), 'low-accuracy' IMU, Sim.run(runs) with Allan() and with
Allan(fit=True), in alternated windows in one process (each arm first in every other window), so that drift of
the shared card's clocks falls on both alike; window 0 warms both arms up and is not counted.  Per window: the wall time of Sim.run and the summed
CUDA-event time of the K13 calls (engine.allan_fit).  K13 alone: CUDA events around engine.allan_fit on 256 x 6
and 100 000 x 6 curves of config 4's grid (model curves with multiplicative scatter, so that every support is
tried), median of 20 launches after 3 warm-up launches.  Prints the card's name and power limit (read in the same
process) and one JSON line per measurement."""
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
from gnss_ins_sim_b200.allan_analysis import Allan  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


class Timer(object):
    """CUDA events around every call of an engine function, summed after a sync."""

    def __init__(self, inner):
        self.inner, self.events = inner, []

    def __call__(self, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = self.inner(*a, **k)
        e1.record()
        self.events.append((e0, e1))
        return out

    def take(self):
        torch.cuda.synchronize()
        t = sum(a.elapsed_time(b) for a, b in self.events) * 1e-3
        self.events = []
        return t


def k13_alone(fit, n, fs, nseries):
    tau = engine.allan_taus(n, fs)
    C = np.array([1e-8, 1e-6, 1e-8, 1e-10, 1e-13])
    model = sum(C[i] * tau ** (i - 2) for i in range(5))
    rng = np.random.default_rng(1)
    var = engine.to_device(model * np.exp(0.3 * rng.standard_normal((nseries, tau.size))))
    for _ in range(3):
        fit(fs, n, var)
    ts = []
    for _ in range(20):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fit(fs, n, var)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    return {'k13_series': nseries, 'ntau': int(tau.size), 'k13_median_s': float(np.median(ts)),
            'k13_min_s': float(np.min(ts)), 'k13_series_per_s': nseries / float(np.median(ts))}


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
    fit = engine.allan_fit
    k13 = engine.allan_fit = Timer(fit)
    arms = (False, True)
    rec = {a: {'wall': [], 'k13': []} for a in arms}
    for w in range(args.windows + 1):
        for arm in (arms if w % 2 == 0 else arms[::-1]):      # either arm first, in turn
            sim = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Allan(fit=arm), seed=seed)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sim.run(args.runs)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            t13 = k13.take()
            if w > 0:
                rec[arm]['wall'].append(dt)
                rec[arm]['k13'].append(t13)
            del sim
    engine.allan_fit = fit
    base, with_fit = float(np.median(rec[False]['wall'])), float(np.median(rec[True]['wall']))
    out = {'config': 4, 'runs': args.runs, 'samples': n, 'allan_windows_s': rec[False]['wall'],
           'allan_fit_windows_s': rec[True]['wall'], 'allan_median_s': base, 'allan_fit_median_s': with_fit,
           'fit_over_plain': with_fit / base, 'k13_in_sim_windows_s': rec[True]['k13'],
           'k13_in_sim_median_s': float(np.median(rec[True]['k13']))}
    lines.append(out)
    print(json.dumps(out), flush=True)
    for nseries in (256 * 6, 100000 * 6):
        r = k13_alone(fit, n, fs, nseries)
        lines.append(r)
        print(json.dumps(r), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'allan_fit_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
