"""K9 (IMU error statistics reduced inside the noise generator) against the unfused alternative, K1 on run
blocks followed by K3p, and against K1 alone, timed with CUDA events.

    python tools/sensor_stats_bench.py [--windows 3] [--block 2000] [--out DIR]

Sizes: 1000 runs x 1000 samples ('mid-accuracy', motion_def-90deg_turn.csv @100 Hz) and 100 000 runs x
193 036 samples ('low-accuracy', motion_def-long_drive.csv @200 Hz, ref_frame 0, BASELINE config 3).  Process
statistics from sample 0.  K1 alone and K1 + K3p write their series into one run block of --block runs
(the whole ensemble is 0.93 TB at config-3 size) and walk the ensemble block by block.  The three variants
are timed in alternated windows; a variant's time is the median of its windows.  Prints the card's name,
power limit and clocks (read in the same process) and one JSON line per size with run-steps/s of each
variant and K9's rate as a share of K1's."""
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
from gnss_ins_sim_b200.sim import trajectory_from_motion_def  # noqa: E402

MOTION = os.path.join(ROOT, 'tests', 'golden')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--windows', type=int, default=3)
    ap.add_argument('--block', type=int, default=2000)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    lines = [{'card': card()}]
    print(json.dumps(lines[0]), flush=True)
    # launches per window: a few hundred milliseconds of GPU time at either size (about 0.1 ms per launch at
    # 1000 x 1000, so that launch overhead and clock ramp-up do not weigh on the ratio)
    for runs, motion, fs, acc, reps in ((1000, 'motion_def-90deg_turn.csv', 100.0, 'mid-accuracy', 2000),
                                        (100000, 'motion_def-long_drive.csv', 200.0, 'low-accuracy', 1)):
        t = trajectory_from_motion_def(fs, os.path.join(MOTION, motion), 0)
        n = t['ref_gyro'].shape[0]
        imu = imu_model.IMU(accuracy=acc, axis=6, gps=False)
        rg, ra = engine.to_device(t['ref_gyro']), engine.to_device(t['ref_accel'])
        blk = min(runs, args.block)

        def k9():
            for _ in range(reps):
                engine.imu_err_stats(fs, runs, rg, ra, imu.gyro_err, imu.accel_err, 1, stats_start=0)

        def k1(reduce):
            def go():
                for _ in range(reps):
                    for r0 in range(0, runs, blk):
                        g, a = engine.imu_noise(fs, min(blk, runs - r0), rg, ra, imu.gyro_err, imu.accel_err, 1,
                                                run_offset=r0)
                        if reduce:
                            engine.proc_stats(g, rg, 0)
                            engine.proc_stats(a, ra, 0)
                        del g, a
            return go

        variants = {'k9': k9, 'k1': k1(False), 'k1_k3p': k1(True)}
        for fn in variants.values():          # warm-up: modules, the allocator's block buffers
            fn()
        torch.cuda.synchronize()
        times = {k: [] for k in variants}
        for _ in range(args.windows):
            for k, fn in variants.items():
                times[k].append(timed(fn) / reps)
        rec = {'runs': runs, 'samples': n, 'accuracy': acc, 'block_runs': blk, 'launch_reps': reps,
               'seconds': times}
        for k in variants:
            rec[k + '_run_steps_per_s'] = runs * n / float(np.median(times[k]))
        rec['k9_share_of_k1_rate'] = rec['k9_run_steps_per_s'] / rec['k1_run_steps_per_s']
        rec['k9_speedup_over_k1_k3p'] = rec['k9_run_steps_per_s'] / rec['k1_k3p_run_steps_per_s']
        lines.append(rec)
        print(json.dumps(rec), flush=True)
        del rg, ra
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'sensor_stats_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
