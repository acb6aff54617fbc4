"""K10 (the magnetometer calibration) timed with CUDA events: the fused form, which regenerates K8's samples in
both passes and writes nothing but 13 values per run, against K8 writing the samples followed by the fed form.

    python tools/magcal_bench.py [--windows 5] [--out DIR]

Two sizes: 100 000 runs x 3 x 1000 samples and 1000 runs x 3 x 60 000 samples, each segment one full rotation
(plus 10 %) of a 47 uT field about one body axis, a 'mid'-grade model (si = I + 0.05 N, hi = 10 uT, std 0.3 uT).
Per size, after one warm-up of each: alternated windows (fused, K8, K8 + fed, fused, ...) of `reps` launches
each between two CUDA events, so that drift of the shared card's clocks falls on all alike; the medians over
windows per launch.  The card's name and power limit are read in the same process.  The fused and the
materialised forms are also checked to agree bit for bit on the timed runs."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import engine  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def rotations(L):
    """ref_mag [3L, 3]: the field rotated once (plus 10 %) about body x, then y, then z; the segments."""
    b = np.array([20.0, -5.0, 42.0])
    ang = np.linspace(0.0, 2.2 * np.pi, L)
    c, s = np.cos(ang), np.sin(ang)
    rows = []
    for i, j in ((1, 2), (2, 0), (0, 1)):
        bb = np.tile(b, (L, 1))
        bb[:, i], bb[:, j] = c * b[i] + s * b[j], -s * b[i] + c * b[j]
        rows.append(bb)
    return np.concatenate(rows), ((0, L), (L, 2 * L), (2 * L, 3 * L))


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--windows', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    lines = [{'card': card()}]
    print(json.dumps(lines[0]), flush=True)
    rng = np.random.default_rng(1)
    err = {'si': np.eye(3) + 0.05 * rng.standard_normal((3, 3)), 'hi': np.array([10.0, -6.0, 3.0]),
           'std': np.full(3, 0.3)}
    for R, L, reps in ((100000, 1000, 3), (1000, 60000, 3)):
        ref, seg = rotations(L)
        ref = engine.to_device(ref)
        n = ref.shape[0]
        state = {}

        def fused():
            state['f'] = engine.mag_calibrate_mc(R, seg, ref, err, 7)

        def k8():
            state['m'] = engine.mag_noise(R, ref, err, 7)

        def fed():
            state['m'] = engine.mag_noise(R, ref, err, 7)
            state['d'] = engine.mag_calibrate(seg, state['m'])

        forms = (('fused', fused), ('k8', k8), ('k8+fed', fed))
        for _, fn in forms:
            fn()
        torch.cuda.synchronize()
        same = (torch.equal(state['f'].soft_iron, state['d'].soft_iron)
                and torch.equal(state['f'].hard_iron, state['d'].hard_iron))
        t = {name: [] for name, _ in forms}
        for _ in range(args.windows):
            for name, fn in forms:
                t[name].append(timed(fn, reps))
        med = {name: float(np.median(v)) for name, v in t.items()}
        rec = {'runs': R, 'samples_per_segment': L, 'run_samples': R * n, 'reps_per_window': reps,
               'windows_s': t, 'median_s': med, 'fused_over_k8': med['fused'] / med['k8'],
               'k8_plus_fed_over_fused': med['k8+fed'] / med['fused'], 'fused_equals_k8_plus_fed': bool(same),
               'fused_run_samples_per_s': R * n / med['fused']}
        lines.append(rec)
        print(json.dumps(rec), flush=True)
        state.clear()
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'magcal_bench.jsonl'), 'w') as f:
            f.write(''.join(json.dumps(x) + '\n' for x in lines))


if __name__ == '__main__':
    main()
