"""K7 on supplied measurements (ekf_kernel<false, true>) against K7 generating its own (ekf_kernel<false, false>),
timed with CUDA events on the same runs.

    python tools/ekf_fed_bench.py [--runs 10000] [--reps 5] [--block 1000] [--out DIR]

Size: BASELINE config 5, motion_def-ins.csv @100 Hz with GPS at 10 Hz (n = 73 250, m = 7 325), demo_ins_loose.py's
IMU, 10 000 runs in one launch.  The fed kernel's inputs are K1's and K6's measurements of the same runs, made in
run blocks of --block runs into one [runs, n, 3] pair and one [runs, m, 6] array (35 GB + 3.5 GB at 10 000 runs),
and it draws the same initial errors, so both kernels filter the same numbers.  The two run in alternated
windows (generated, fed, generated, ...), one launch per window, so that drift of the shared card's clocks falls
on both alike.  Prints the card's name and power limit (read in the same process) and one JSON line per kernel:
median time, run-steps/s and, for the fed kernel, the bytes it must read (48 B per run-sample of IMU, 48 B per
run-row of GPS) per second against the H100 SXM's 3.35 TB/s; and the largest end-point difference of the two."""
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
HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet (700 W card)


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
    ap.add_argument('--block', type=int, default=1000)
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
    d, n, runs, fs, seed = sim._dev, sim._traj['ref_gyro'].shape[0], args.runs, 100.0, 5
    m = d['ref_gps'].shape[0]
    ini = sim._traj['ini']
    gyro = torch.empty((runs, n, 3), dtype=torch.float64, device='cuda')
    accel = torch.empty_like(gyro)
    gps = torch.empty((runs, m, 6), dtype=torch.float64, device='cuda')
    for r0 in range(0, runs, args.block):
        r1 = min(runs, r0 + args.block)
        g, a = engine.imu_noise(fs, r1 - r0, d['ref_gyro'], d['ref_accel'], imu.gyro_err, imu.accel_err, seed,
                                run_offset=r0)
        gyro[r0:r1], accel[r0:r1] = g, a
        gps[r0:r1] = engine.gps_noise(r1 - r0, d['ref_gps'], imu.gps_err, 0, seed, run_offset=r0)
        del g, a
    torch.cuda.synchronize()
    out = {}

    def launch(kind):
        if kind == 'generated':
            out[kind] = engine.ins_loose(fs, runs, seed, imu.gyro_err, imu.accel_err, imu.gps_err, ini,
                                         d['ref_gyro'], d['ref_accel'], d['ref_nav'], d['ref_gps'], d['gps_idx'],
                                         d['gps_vis'], stats_start=3000, out=out.get(kind))
        else:
            out[kind] = engine.ins_loose_fed(fs, gyro, accel, gps, d['gps_idx'], d['gps_vis'], imu.gyro_err,
                                             imu.accel_err, imu.gps_err, ini, seed=seed, ini_draw=True,
                                             ref_nav=d['ref_nav'], out=out.get(kind))
    kinds = ('generated', 'fed')
    for kind in kinds:                       # warm-up, and the result buffers of both
        launch(kind)
    torch.cuda.synchronize()
    diff = {k: float((out['fed'].__dict__[k] - out['generated'].__dict__[k]).abs().max())
            for k in ('end_err', 'end_bias')}
    ms = {kind: [] for kind in kinds}
    for _ in range(args.reps):
        for kind in kinds:
            ms[kind].append(timed(lambda: launch(kind)))
    base = float(np.median(ms['generated']))
    for kind in kinds:
        med = float(np.median(ms[kind]))
        rec = {'kernel': 'K7 ekf_kernel<false, %s>' % ('true' if kind == 'fed' else 'false'), 'measurements': kind,
               'runs': runs, 'samples': n, 'gps_rows': m, 'ms': ms[kind], 'median_ms': med,
               'ratio_to_generated': med / base, 'run_steps_per_s': runs * n / (med * 1e-3)}
        if kind == 'fed':
            nbytes = runs * (n * 48 + m * 48)
            rec.update(bytes_read=nbytes, bytes_per_s=nbytes / (med * 1e-3),
                       share_of_3_35_TBps=nbytes / (med * 1e-3) / HBM_BYTES_PER_S,
                       max_abs_diff_to_generated=diff)
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'ekf_fed_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
