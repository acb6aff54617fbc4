"""K7 (the loosely-coupled filter, ekf_kernel) without and with a run-to-run turn-on bias, timed with CUDA events.

    python tools/ekf_runerr_bench.py [--runs 10000] [--reps 5] [--out DIR]

Size: BASELINE config 5, motion_def-ins.csv @100 Hz with GPS at 10 Hz (n = 73 250), demo_ins_loose.py's IMU,
10 000 runs in one launch.  'plain' is that IMU through today's kernel (ekf_kernel<false, false, false>); 'rb' adds
gyro_b_std 10 deg/h and accel_b_std 5e-4 m/s^2 and asks for the bias-estimate errors, which launches the RB form
(ekf_kernel<false, false, false, false, true>: one prologue draw per channel, six more quad shuffles per GPS epoch
and six at the end).  After a warm-up of each, the two run in alternated windows (plain, rb, plain, ...), so that
drift of the shared card's clocks falls on both alike; every window is one launch.  Prints the card's name and
power limit (read in the same process) and one JSON line per form with its median time and its ratio to plain."""
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
TURN_ON = {'gyro_b_std': np.full(3, 10.0), 'accel_b_std': np.full(3, 5e-4)}


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
    imus = {'plain': imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True),
            'rb': imu_model.IMU(accuracy=dict(DEMO_IMU, **TURN_ON), axis=6, gps=True)}
    sim = Sim([100.0, 10.0, 0.0], os.path.join(ROOT, 'tests', 'golden', 'motion_def-ins.csv'), ref_frame=0,
              imu=imus['plain'], algorithm=InsLoose(), seed=5)
    sim.run(8)                               # the trajectory and its device copies
    d, n, runs, fs = sim._dev, sim._traj['ref_gyro'].shape[0], args.runs, 100.0
    out = {}

    def launch(kind):
        imu = imus[kind]
        out[kind] = engine.ins_loose(fs, runs, 5, imu.gyro_err, imu.accel_err, imu.gps_err, sim._traj['ini'],
                                     d['ref_gyro'], d['ref_accel'], d['ref_nav'], d['ref_gps'], d['gps_idx'],
                                     d['gps_vis'], stats_start=3000, bias_err=kind == 'rb', out=out.get(kind))
    for kind in imus:                        # warm-up, and the result buffers of both forms
        launch(kind)
    torch.cuda.synchronize()
    ms = {kind: [] for kind in imus}
    for _ in range(args.reps):
        for kind in imus:
            ms[kind].append(timed(lambda: launch(kind)))
    base = float(np.median(ms['plain']))
    for kind in imus:
        med = float(np.median(ms[kind]))
        rec = {'kernel': 'K7 ekf_kernel<false, false, false%s>' % (', false, true' if kind == 'rb' else ''),
               'form': kind, 'runs': runs, 'samples': n, 'ms': ms[kind], 'median_ms': med, 'ratio_to_plain': med / base,
               'run_steps_per_s': runs * n / (med * 1e-3)}
        if kind == 'rb':
            c = out[kind].consist.cpu().numpy()
            ep = np.maximum(c[:, 18:19], 1.0)
            rec['mean_nees'] = (c[:, 0:3] / ep).mean(0).tolist()
            rec['min_inside3'] = float((c[:, 3:18] / ep).mean(0).min())
            sig = np.concatenate([imus['rb'].gyro_err['b_std'], imus['rb'].accel_err['b_std']])
            rec['bias_err_std_over_b_std'] = (out[kind].end_bias_err.cpu().numpy().std(0) / sig).tolist()
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'ekf_runerr_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
