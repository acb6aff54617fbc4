"""K7 (the loosely-coupled filter, ekf_kernel) with and without process-error statistics, timed with CUDA events.

    python tools/ekf_proc_bench.py [--runs 10000] [--reps 5] [--out DIR]

Size: BASELINE config 5, motion_def-ins.csv @100 Hz with GPS at 10 Hz (n = 73 250), demo_ins_loose.py's IMU,
10 000 runs in one launch, no vibration.  Variants: no statistics (ekf_kernel<false, false, false>), and
statistics from sample 0 (ekf_kernel<false, false, true>) with the position in LLA, NED and ECEF.  They run in
alternated windows (none, LLA, NED, ECEF, none, ...), so that drift of the shared card's clocks falls on all of
them alike; every window is one launch.  Prints the card's name and power limit (read in the same process) and
one JSON line per variant with its median time and its ratio to no statistics."""
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
    variants = {'none': None, 'lla': engine.POS_FRAME_LLA, 'ned': engine.POS_FRAME_NED,
                'ecef': engine.POS_FRAME_ECEF}
    out = {}

    def launch(kind):
        frame = variants[kind]
        out[kind] = engine.ins_loose(fs, runs, 5, imu.gyro_err, imu.accel_err, imu.gps_err, sim._traj['ini'],
                                     d['ref_gyro'], d['ref_accel'], d['ref_nav'], d['ref_gps'], d['gps_idx'],
                                     d['gps_vis'], stats_start=3000, proc_start=None if frame is None else 0,
                                     proc_pos_frame=frame or 0, out=out.get(kind))
    for kind in variants:                    # warm-up, and the result buffers of every variant
        launch(kind)
    torch.cuda.synchronize()
    # the statistics change nothing else the filter computes
    same = all(torch.equal(getattr(out[k], a), getattr(out['none'], a)) for k in variants
               for a in ('end_err', 'end_bias', 'consist'))
    ms = {kind: [] for kind in variants}
    for _ in range(args.reps):
        for kind in variants:
            ms[kind].append(timed(lambda: launch(kind)))
    base = float(np.median(ms['none']))
    for kind in variants:
        med = float(np.median(ms[kind]))
        rec = {'kernel': 'K7 ekf_kernel<false, false, %s>' % ('false' if kind == 'none' else 'true'),
               'proc_stats': kind, 'runs': runs, 'samples': n, 'ms': ms[kind], 'median_ms': med,
               'ratio_to_none': med / base, 'added_us_per_step': (med - base) * 1e3 / n,
               'other_outputs_bit_identical': same}
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'ekf_proc_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
