"""K7 (the loosely-coupled filter, ekf_kernel) with and without vibration, timed with CUDA events.

    python tools/ekf_vib_bench.py [--runs 10000] [--reps 5] [--out DIR]

Size: BASELINE config 5, motion_def-ins.csv @100 Hz with GPS at 10 Hz (n = 73 250), demo_ins_loose.py's IMU,
10 000 runs in one launch.  Vibration: none, random (0.05 g, 0.5 deg/s), sinusoidal (0.05 g at 7.5 Hz,
0.5 deg/s at 3 Hz) and PSD (K5 series of all runs, made once and timed on their own).  The four K7 variants
run in alternated windows (none, random, sinusoidal, PSD, none, ...), so that drift of the shared card's
clocks falls on all of them alike; every window is one launch.  Prints the card's name and power limit (read
in the same process) and one JSON line per variant with its median time and its ratio to no vibration."""
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
from gnss_ins_sim_b200.sim import Sim, parse_env  # noqa: E402

DEMO_IMU = {'gyro_b': np.zeros(3), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
            'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
            'accel_b': np.zeros(3), 'accel_vrw': np.array([0.03119, 0.03009, 0.04779]),
            'accel_b_stability': np.array([4.29e-5, 5.72e-5, 8.02e-5]),
            'accel_b_corr': np.array([200.0, 200.0, 200.0])}       # demo_ins_loose.py:28-37
PSD = np.stack([np.linspace(0.0, 50.0, 26), np.full(26, 1e-2), np.linspace(1e-2, 4e-2, 26),
                np.full(26, 2e-2)], axis=1)


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
    psd = parse_env(PSD, fs), parse_env(PSD * 1e-4, fs)
    k5_ms = []

    def make_series():
        return [engine.psd_series(fs, n, runs, sensor, v, 5) for sensor, v in ((0, psd[0]), (1, psd[1]))]
    make_series()                            # warm-up
    torch.cuda.synchronize()
    for _ in range(args.reps):
        k5_ms.append(timed(make_series))
    (sa, na), (sg, ng) = make_series()
    variants = {'none': (None, None),
                'random': (parse_env('[0.05 0.05 0.05]g-random', fs), parse_env('[0.5 0.5 0.5]d-random', fs)),
                'sinusoidal': (parse_env('[0.05 0.05 0.05]g-7.5Hz-sinusoidal', fs),
                               parse_env('[0.5 0.5 0.5]d-3Hz-sinusoidal', fs)),
                'psd': (engine.vib_series(sa, na), engine.vib_series(sg, ng))}
    out = {}

    def launch(kind):
        va, vg = variants[kind]
        out[kind] = engine.ins_loose(fs, runs, 5, imu.gyro_err, imu.accel_err, imu.gps_err, sim._traj['ini'],
                                     d['ref_gyro'], d['ref_accel'], d['ref_nav'], d['ref_gps'], d['gps_idx'],
                                     d['gps_vis'], stats_start=3000, vib_accel=va, vib_gyro=vg,
                                     out=out.get(kind))
    for kind in variants:                    # warm-up, and the result buffers of every variant
        launch(kind)
    torch.cuda.synchronize()
    ms = {kind: [] for kind in variants}
    for _ in range(args.reps):
        for kind in variants:
            ms[kind].append(timed(lambda: launch(kind)))
    base = float(np.median(ms['none']))
    for kind in variants:
        med = float(np.median(ms[kind]))
        rec = {'kernel': 'K7 ekf_kernel<%s>' % ('false' if kind == 'none' else 'true'), 'vibration': kind,
               'runs': runs, 'samples': n, 'ms': ms[kind], 'median_ms': med, 'ratio_to_none': med / base,
               'run_steps_per_s': runs * n / (med * 1e-3)}
        if kind == 'psd':
            rec['k5_psd_series_ms_both_sensors'] = k5_ms
            rec['k5_median_ms'] = float(np.median(k5_ms))
            rec['series_bytes'] = int(sa.numel() + sg.numel()) * 8
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'ekf_vib_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
