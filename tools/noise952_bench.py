"""What the IEEE Std 952 terms cost: K1 and K9 with and without them, and free integration through K1 then K2
against the fused Monte-Carlo kernel (K12).

    python tools/noise952_bench.py [--windows 5] [--k1-runs 16]

K1 / K9 at config 4's shape (static 10 h @400 Hz, n = 14.4 M samples, 'low-accuracy' IMU): K9 on 256 runs (it
materialises nothing), K1 on --k1-runs runs (256 runs of materialised series would need 177 GB).  The terms arm
sets every term of both sensors (q, rrw, rr), the ramp arm only rr (the ex kernels, without a walk or quantisation
draw); the plain arm runs the plain kernels.  CUDA events around each call.  Config 2 (motion_def-90deg_turn, n = 1000 @100 Hz,
'mid-accuracy', 1000 runs, Sim.run + get_error_stats('pos')): the K12 route against the K1 -> K2 route, forced
with Sim's private switch (the IMU without terms, so both compute the same numbers), host wall clock with a
device synchronise.  Window 0 warms every arm up and is not counted; the arms alternate which goes first.
Prints the card's name and power limit (read in the same process) and one JSON line per measurement: medians
over the windows."""
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
from gnss_ins_sim_b200.free_integration import FreeIntegration  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def events(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    del out
    return e0.elapsed_time(e1) * 1e-3


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def alternate(arms, windows, clock):
    """{name: median seconds} over windows 1..windows-1, each arm first in alternate windows."""
    names = list(arms)
    got = {k: [] for k in names}
    for w in range(windows):
        for k in (names if w % 2 == 0 else names[::-1]):
            t = clock(arms[k])
            if w:
                got[k].append(t)
    return {k: float(np.median(v)) for k, v in got.items()}, got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--windows', type=int, default=5)
    ap.add_argument('--k1-runs', type=int, default=16)
    args = ap.parse_args()
    print(json.dumps({'card': card()}))
    n, fs = 14400000, 400.0
    plain = imu_model.IMU('low-accuracy', gps=False)
    terms = imu_model.IMU('low-accuracy', gps=False)
    terms.set_gyro_error({'q': np.full(3, 1e-6), 'rrw': np.full(3, 2e-6), 'rr': np.full(3, 1e-7)})
    terms.set_accel_error({'q': np.full(3, 1e-4), 'rrw': np.full(3, 1e-4), 'rr': np.full(3, 1e-6)})
    ramp = imu_model.IMU('low-accuracy', gps=False)       # a ramp alone: the ex kernels make no extra draw
    ramp.set_gyro_error({'rr': np.full(3, 1e-7)})
    ramp.set_accel_error({'rr': np.full(3, 1e-6)})
    rg = engine.to_device(np.zeros((n, 3)))
    ra = engine.to_device(np.tile(np.array([4.9, 0.0, -8.487]), (n, 1)))

    def k1(imu):
        return lambda: engine.imu_noise(fs, args.k1_runs, rg, ra, imu.gyro_err, imu.accel_err, 1)

    def k9(imu):
        return lambda: engine.imu_err_stats(fs, 256, rg, ra, imu.gyro_err, imu.accel_err, 1, stats_start=0)

    for name, mk, runs in (('K1', k1, args.k1_runs), ('K9', k9, 256)):
        med, raw = alternate({'plain': mk(plain), 'terms': mk(terms), 'ramp': mk(ramp)}, args.windows, events)
        print(json.dumps({'kernel': name, 'runs': runs, 'samples': n, 'seconds_median': med,
                          'terms_over_plain': med['terms'] / med['plain'],
                          'ramp_over_plain': med['ramp'] / med['plain'],
                          'run_samples_per_s': {k: runs * n / v for k, v in med.items()},
                          'windows': raw}))
    del rg, ra
    torch.cuda.empty_cache()
    g = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'traj_90deg_turn_100hz_rf1.npz')))
    traj = {k: g[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    mid = imu_model.IMU('mid-accuracy', gps=False)

    def config2(fed):
        def go():
            sim = Sim([100.0, 0.0, 0.0], traj, ref_frame=1, imu=mid, algorithm=FreeIntegration(g['ini']), seed=12345)
            sim._force_fed = fed
            sim.run(1000)
            sim.get_error_stats('pos', err_stats_start=-1)
        return go

    med, raw = alternate({'K12': config2(False), 'K1_K2': config2(True)}, args.windows + 2, wall)
    print(json.dumps({'workload': 'config 2 Sim.run(1000) + get_error_stats', 'seconds_median': med,
                      'k1_k2_over_k12': med['K1_K2'] / med['K12'], 'windows': raw}))


if __name__ == '__main__':
    main()
