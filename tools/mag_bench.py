"""K8 (magnetometer measurement generator, mag_noise_kernel) timed with CUDA events over many launches.

    python tools/mag_bench.py [--reps 5] [--out DIR]

Sizes: 1000 runs x 1000 samples (motion_def-90deg_turn.csv @100 Hz) and 1000 runs x 193 036 samples
(motion_def-long_drive.csv @200 Hz, BASELINE config 3's length).  Per size: units (run-samples) per second,
bytes written per second against the H100 SXM's 3.35 TB/s HBM3, and the kernel's FP64 instruction issue
against the card's measured FP64 FMA issue rate (b2ins_diag_dfma_rate), from the FP64 instructions per
unit counted in the kernel's SASS (cuobjdump).  The larger of the two shares names the bound it sits
nearer.  Prints the card's name and power limit (read in the same process) and one JSON line per size."""
import argparse
import ctypes
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import _lib, engine  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
KERNEL = '_ZN5b2ins16mag_noise_kernelENS_9MagParamsE'


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def sass_counts():
    """Static instruction counts of the kernel's SASS: all, FP64 (D* arithmetic and 64-bit MUFU / F2F / I2F)."""
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    res = subprocess.run([exe, '-sass', _lib.lib_path()], capture_output=True, text=True)
    body, on = [], False
    for line in res.stdout.splitlines():
        if 'Function : ' in line:
            on = line.strip().endswith(KERNEL)
        elif on:
            m = re.match(r'\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)', line)
            if m:
                body.append(m.group(1))
    fp64 = [op for op in body if re.match(r'D(FMA|MUL|ADD|SETP|MNMX)', op) or
            (op.startswith(('MUFU', 'F2F', 'I2F', 'F2I')) and '64' in op)]
    return {'instructions': len(body), 'fp64': len(fp64),
            'fp64_by_op': {op: fp64.count(op) for op in sorted(set(fp64))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    lines = [{'card': card()}]
    print(json.dumps(lines[0]), flush=True)
    rate = ctypes.c_double(0.0)
    _lib.check(_lib.load().b2ins_diag_dfma_rate(ctypes.byref(rate)))
    sass = sass_counts()
    lines.append({'dfma_per_s': rate.value, 'sass': sass})
    print(json.dumps(lines[-1]), flush=True)
    err = {'si': np.array([[1.02, 0.03, -0.01], [-0.02, 0.97, 0.05], [0.04, -0.06, 1.01]]),
           'hi': np.array([10.0, -7.5, 3.0]), 'std': np.array([0.2, 0.35, 0.5])}
    rng = np.random.default_rng(1)
    lib = _lib.load()
    si, hi, std = (np.ascontiguousarray(err[k], dtype=np.float64) for k in ('si', 'hi', 'std'))
    for runs, n, per_window in ((1000, 1000, 200), (1000, 193036, 5)):
        ref = engine.to_device(rng.standard_normal((n, 3)) * 30.0)
        out = torch.empty((runs, n, 3), dtype=torch.float64, device='cuda')

        def launch():
            _lib.check(lib.b2ins_mag_noise_f64(runs, n, engine._ptr(ref), _lib.host_ptr(si), _lib.host_ptr(hi),
                                               _lib.host_ptr(std), 3, 0, engine._ptr(out), engine._stream()))
        # the launches of a window are replayed from a CUDA graph, so that the host's enqueue rate
        # (a few microseconds per ctypes call) does not pace the 1000 x 1000 size
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            launch()                                      # warm-up
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(per_window):
                launch()
        graph.replay()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1) / per_window)
        del graph, out
        t = float(np.median(ms)) * 1e-3
        units = runs * n
        rec = {'runs': runs, 'samples': n, 'launches_per_window': per_window, 'ms_per_launch': ms,
               'median_ms': t * 1e3, 'units_per_s': units / t,
               'write_GB_per_s': 24.0 * units / t / 1e9, 'hbm_write_share': 24.0 * units / t / HBM_BYTES_PER_S,
               'fp64_instr_per_unit': sass['fp64'],
               'fp64_issue_share': sass['fp64'] * units / t / rate.value}
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'mag_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
