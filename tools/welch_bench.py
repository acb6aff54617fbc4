"""Welch spectra (K11) of BASELINE config 4 through Sim, with a torch.fft baseline on the same device blocks.

    python tools/welch_bench.py [--runs 256] [--windows 3] [--out DIR]

Config 4: static 10 h @400 Hz (n = 14.4 M samples), 'low-accuracy' IMU, Sim.run(runs) with Psd(nperseg=16384) and
with Psd(nperseg=256), in alternated windows in one process, so that drift of the shared card's clocks falls on
both alike.  Sim materialises K1's series in run blocks and hands each block to K11.  Per window: the wall time of
Sim.run, and the summed CUDA-event time of the K11 calls (engine.welch) and of K1's materialisation
(engine.imu_noise).  K11's bytes and FP64 operations are counted from shapes: every sample is read from HBM once
(8 B per series-sample; the overlap of adjacent segments comes from L2), and a segment costs 5 M log2 M for the
length-M complex transform (10 operations per radix-2 butterfly), 30 per bin for the split and |X|^2 and 3 per
sample for the mean, the window and the packing.  The share of peak is the larger of the HBM bound (3.35 TB/s,
the H100 SXM data sheet) and the FP64 bound (2 operations per DFMA at the rate b2ins_diag_dfma_rate measures)
over K11's time.  Baseline, for comparison only: the first window also sends every block through torch.fft.rfft
on unfolded, detrended, windowed segments (CUDA events around it).  Prints the card's name and power limit (read
in the same process) and one JSON line per nperseg with medians."""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import _lib, engine, imu_model  # noqa: E402
from gnss_ins_sim_b200.sim import Sim  # noqa: E402
from gnss_ins_sim_b200.psd_analysis import Psd  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def torch_welch(x, nseries, n, N, D, window, inner, outer_stride, sample_stride):
    """The same spectra with torch.fft.rfft, without the 1/fs: [nseries, L].  Eight series at a time, so that the
    unfolded segments (twice the series at 50 % overlap) fit beside Sim's run block."""
    if inner == 1:
        s = x.reshape(-1)[:nseries * n].reshape(nseries, n)
    else:
        s = x.reshape(-1, n, inner).permute(0, 2, 1).reshape(-1, n)
    out = []
    for i in range(0, nseries, 8):
        seg = s[i:i + 8].unfold(1, N, N - D)
        seg = seg - seg.mean(dim=2, keepdim=True)
        p = torch.fft.rfft(seg * window, dim=2).abs().square_().mean(dim=1)
        p[:, 1:-1] *= 2.0
        out.append(p / window.square().sum())
    return torch.cat(out)


class Timer(object):
    """CUDA events around every call of an engine function, summed after a sync."""

    def __init__(self, inner, baseline=None):
        self.inner, self.baseline = inner, baseline
        self.events, self.base_events, self.series_samples = [], [], 0
        self.run_baseline = False

    def __call__(self, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = self.inner(*a, **k)
        e1.record()
        self.events.append((e0, e1))
        if self.baseline is not None:
            fs, x, n, nseries = a[:4]
            self.series_samples += n * nseries
            if self.run_baseline:
                b0, b1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                N, D, w = a[4], a[5], engine.to_device(a[6], x.device)
                b0.record()
                ref = self.baseline(x, nseries, n, N, D, w, k.get('inner', 1), None, k.get('sample_stride', 1))
                b1.record()
                self.base_events.append((b0, b1))
                self.max_rel = max(getattr(self, 'max_rel', 0.0),
                                   float(((out[0] - ref / a[0]).abs() / ref.div(a[0]).abs().amax()).max()))
        return out

    def take(self):
        torch.cuda.synchronize()
        t = sum(a.elapsed_time(b) for a, b in self.events) * 1e-3
        tb = sum(a.elapsed_time(b) for a, b in self.base_events) * 1e-3
        ss = self.series_samples
        self.events, self.base_events, self.series_samples = [], [], 0
        return t, tb, ss


def fp64_ops(series_samples, n, N, D):
    K = (n - D) // (N - D)
    M = N // 2
    per_seg = 5 * M * math.log2(M) + 30 * (M + 1) + 3 * N
    return series_samples / n * K * per_seg


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
    dfma = ctypes.c_double(0.0)
    _lib.check(_lib.load().b2ins_diag_dfma_rate(ctypes.byref(dfma)))
    n, fs, seed = 14400000, 400.0, 5
    traj = {'ref_pos': np.zeros((n, 3)), 'ref_vel': np.zeros((n, 3)), 'ref_att': np.zeros((n, 3)),
            'ref_accel': np.tile(np.array([4.9, 0.0, -8.487]), (n, 1)), 'ref_gyro': np.zeros((n, 3))}
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    k11 = engine.welch = Timer(engine.welch, torch_welch)
    k1 = engine.imu_noise = Timer(engine.imu_noise)
    arms = (16384, 256)
    rec = {N: {'wall': [], 'k11': [], 'k1': [], 'torch': None, 'ss': 0} for N in arms}
    for w in range(args.windows + 1):          # window 0 warms up both arms and runs the torch.fft baseline
        for N in arms:
            sim = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Psd(nperseg=N), seed=seed)
            k11.run_baseline = (w == 0)
            k11.max_rel = 0.0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sim.run(args.runs)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            t11, tb, ss = k11.take()
            t1, _, _ = k1.take()
            if w == 0:
                rec[N]['torch'], rec[N]['torch_max_rel_diff'] = tb, k11.max_rel
            else:
                rec[N]['wall'].append(dt)
                rec[N]['k11'].append(t11)
                rec[N]['k1'].append(t1)
                rec[N]['ss'] = ss
            del sim
    for N in arms:
        r = rec[N]
        t = float(np.median(r['k11']))
        ss = r['ss']
        hbm = 8 * ss
        ops = fp64_ops(ss, n, N, N // 2)
        t_hbm, t_fp64 = hbm / HBM_BYTES_PER_S, ops / (2 * dfma.value)
        out = {'nperseg': N, 'runs': args.runs, 'samples': n, 'series_samples': ss,
               'sim_run_windows_s': r['wall'], 'sim_run_median_s': float(np.median(r['wall'])),
               'k11_windows_s': r['k11'], 'k11_median_s': t, 'k1_windows_s': r['k1'],
               'k1_median_s': float(np.median(r['k1'])),
               'k11_hbm_bytes': hbm, 'k11_fp64_ops': ops, 'k11_fp64_ops_per_s': ops / t,
               'dfma_per_s': dfma.value, 'bound': 'hbm' if t_hbm >= t_fp64 else 'fp64',
               'k11_share_of_peak': max(t_hbm, t_fp64) / t,
               'torch_fft_s': r['torch'], 'torch_fft_max_rel_diff': r['torch_max_rel_diff'],
               'k11_over_torch_fft': t / r['torch'] if r['torch'] else None}
        lines.append(out)
        print(json.dumps(out), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'welch_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
