"""K7 (the loosely-coupled filter, ekf_kernel) with and without alignment, timed with CUDA events.

    python tools/ekf_align_bench.py [--runs 10000] [--reps 5] [--out DIR]

Size: BASELINE config 5, motion_def-ins.csv @100 Hz with GPS at 10 Hz (n = 73 250), demo_ins_loose.py's IMU,
10 000 runs in one launch, no vibration.  Variants: the filter from the truth plus the P0 draw
(b2ins_ins_loose_ex_f64, align off) and the self-initialising filter with a given heading and with the GPS
heading (b2ins_ins_loose_align_f64, the same instantiation with EkfParams::align set).  They run in alternated
windows (off, yaw, gps, off, ...), so that drift of the shared card's clocks falls on all of them alike; every
window is one launch.  Prints the card's name and power limit (read in the same process) and one JSON line per
variant with its median time and its ratio to align off."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import engine, imu_model  # noqa: E402
from gnss_ins_sim_b200.ins_loose import InsLoose  # noqa: E402
from gnss_ins_sim_b200.sim import Sim  # noqa: E402

DEMO_IMU = {'gyro_b': np.zeros(3), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
            'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
            'accel_b': np.zeros(3), 'accel_vrw': np.array([0.03119, 0.03009, 0.04779]),
            'accel_b_stability': np.array([4.29e-5, 5.72e-5, 8.02e-5]),
            'accel_b_corr': np.array([200.0, 200.0, 200.0])}       # demo_ins_loose.py:28-37


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=10000)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    lines = [{'card': card()}]
    print(json.dumps(lines[0]), flush=True)
    imu = imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True)
    sim = Sim([100.0, 10.0, 0.0], os.path.join(ROOT, 'tests', 'golden', 'motion_def-ins.csv'), ref_frame=0,
              imu=imu, algorithm=InsLoose(), seed=5)
    sim.run(8)                               # the trajectory and its device copies
    d, n, runs, fs = sim._dev, sim._traj['ref_gyro'].shape[0], args.runs, 100.0
    # motion_def-ins.csv starts at rest: the GPS heading needs motion, so its variant fixes on a moving epoch
    gps_vis_moving = d['gps_vis'].clone()
    gps_vis_moving[:3000] = 0.0              # 300 s, after the first acceleration
    variants = {'off': None, 'yaw': (0.1, 0.15 ** 2), 'gps': ('gps', 0.0)}
    out = {}

    def launch(kind):
        vis = gps_vis_moving if kind == 'gps' else d['gps_vis']
        out[kind] = engine.ins_loose(fs, runs, 5, imu.gyro_err, imu.accel_err, imu.gps_err, sim._traj['ini'],
                                     d['ref_gyro'], d['ref_accel'], d['ref_nav'], d['ref_gps'], d['gps_idx'], vis,
                                     stats_start=3000, out=out.get(kind), align=variants[kind])
    for kind in variants:                    # warm-up, and the result buffers of every variant
        launch(kind)
    torch.cuda.synchronize()
    finite = {k: bool(torch.isfinite(out[k].end_err).all()) for k in variants}
    ms = {kind: [] for kind in variants}
    for _ in range(args.reps):
        for kind in variants:
            ms[kind].append(timed(lambda: launch(kind)))
    base = float(np.median(ms['off']))
    for kind in variants:
        med = float(np.median(ms[kind]))
        rec = {'kernel': 'K7 ekf_kernel<false, false, false>', 'align': kind, 'fix_sample': out[kind].start,
               'runs': runs, 'samples': n, 'ms': ms[kind], 'median_ms': med, 'ratio_to_off': med / base,
               'end_err_finite': finite[kind]}
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'ekf_align_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
