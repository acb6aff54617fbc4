"""Cost of NED / ECEF process-error statistics: the PROC launch of the fused Monte-Carlo kernel (ref_frame 0,
'low-accuracy' IMU, stats_start 0) with the position columns in LLA (proc_pos_frame 0) against NED (1), timed
with CUDA events, the two frames alternated in one process.

    python tools/proc_frame_bench.py [--sizes small,c3] [--reps 5]

small: 1000 runs x 1000 samples (tests/golden/traj_90deg_turn_100hz_rf0.npz), 20 launches per timing window.
c3:    BASELINE config 3's size, 100 000 runs x 193 036 samples (motion_def-long_drive.csv @200 Hz), one launch
       per window.
Prints the card's name and power limit and one JSON line per size."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import engine, imu_model, pathgen  # noqa: E402
from gnss_ins_sim_b200.sim import trajectory_from_motion_def  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def workload(size):
    if size == 'small':
        g = np.load(os.path.join(ROOT, 'tests', 'golden', 'traj_90deg_turn_100hz_rf0.npz'))
        traj, fs, runs, ini, per_window = {k: g[k] for k in g.files}, float(g['fs']), 1000, g['ini'], 20
    else:
        csv = os.path.join(ROOT, 'tests', 'golden', 'motion_def-long_drive.csv')
        traj, fs, runs, ini, per_window = trajectory_from_motion_def(200.0, csv, 0), 200.0, 100000, \
            pathgen.parse_motion(csv)[0], 1
    nav = np.ascontiguousarray(np.concatenate([traj['ref_att'], traj['ref_pos'], traj['ref_vel']], axis=1))
    dev = [engine.to_device(a) for a in (traj['ref_gyro'], traj['ref_accel'], nav, np.asarray(ini)[None])]
    return dev, fs, traj['ref_gyro'].shape[0], runs, per_window


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='small,c3')
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    print(json.dumps({'card': card()}), flush=True)
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    for size in args.sizes.split(','):
        dev, fs, n, runs, per_window = workload(size)
        cfg = {f: engine.make_mc_config(0, fs, n, runs, 3, imu.gyro_err, imu.accel_err, 1, 9, stats_start=0,
                                        proc_pos_frame=f) for f in (0, 1)}
        out = {f: engine.mc_free_integration(cfg[f], *dev) for f in (0, 1)}    # warm-up, and the outputs
        torch.cuda.synchronize()
        ps = {f: out[f].proc_stats.cpu().numpy() for f in (0, 1)}
        same = bool(np.array_equal(ps[0][:, :, 0:3], ps[1][:, :, 0:3]) and
                    np.array_equal(ps[0][:, :, 6:9], ps[1][:, :, 6:9]))
        ms = {0: [], 1: []}
        for rep in range(args.reps):
            for f in ((0, 1) if rep % 2 == 0 else (1, 0)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(per_window):
                    engine.mc_free_integration(cfg[f], *dev, out=out[f])
                e1.record()
                torch.cuda.synchronize()
                ms[f].append(e0.elapsed_time(e1) / per_window)
        print(json.dumps({'size': size, 'runs': runs, 'samples': n, 'lanes_per_run': 'auto',
                          'ms_per_launch_lla': ms[0], 'ms_per_launch_ned': ms[1],
                          'median_lla_ms': float(np.median(ms[0])), 'median_ned_ms': float(np.median(ms[1])),
                          'ned_over_lla': float(np.median(ms[1]) / np.median(ms[0])),
                          'att_vel_columns_equal': same,
                          'ned_pos_std_m_run0': ps[1][0, 2, 3:6].tolist()}), flush=True)


if __name__ == '__main__':
    main()
