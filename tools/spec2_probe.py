"""Sweep of the warp-specialised K12 shapes (mc_spec_kernel.cuh): run-steps/s for
(runs, lanes per run G, producers per integrator P, integrator warps per CTA WI, split) on the
config-2 trajectory (n = 1000) in both frames.  GPU box only; one JSON line per point.
    python tools/spec2_probe.py [quick]"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import engine  # noqa: E402

MID_G = {'b': np.zeros(3), 'b_drift': np.full(3, 3.5 * np.pi / 180 / 3600),
         'b_corr': np.full(3, 100.0), 'arw': np.full(3, 0.25 * np.pi / 180 / 60)}
MID_A = {'b': np.zeros(3), 'b_drift': np.full(3, 5e-5), 'b_corr': np.full(3, 100.0),
         'vrw': np.full(3, 0.03 / 60)}
SHAPES = {1: ['3,1,0', '6,1,0', '0'], 2: ['3,1,0', '6,1,0'], 4: ['3,1,0', '6,1,0', '6,1,1', '6,2,0'], 8: ['6,1,0', '6,2,0'],
          16: ['1,4,0', '1,4,1'], 32: ['1,4,1']}


def main():
    quick = len(sys.argv) > 1 and sys.argv[1] == 'quick'
    sweeps = [(1000, [4, 8, 16, 32, 2]), (500, [4, 8, 16]), (2000, [2, 4, 1]), (4000, [1, 2, 4]),
              (8000, [1, 2]), (12500, [1, 2, 4]), (40000, [1, 2]), (65536, [1]), (100000, [1]),
              (262144, [1]), (1000000, [1])]
    if quick:
        sweeps = [(1000, [4, 8]), (500, [8, 4]), (2000, [4, 2])]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    for rf in (1, 0):
        g = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'traj_90deg_turn_100hz_rf%d.npz' % rf)))
        nav = np.concatenate([g['ref_att'], g['ref_pos'], g['ref_vel']], axis=1)
        n = nav.shape[0]
        dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda()
               for a in (g['ref_gyro'], g['ref_accel'], nav, g['ini'][None])]
        for R, lanes_list in sweeps:
            for lanes in lanes_list:
                for shape in SHAPES[lanes]:
                    os.environ['B2INS_MC_SHAPE'] = shape
                    cfg = engine.make_mc_config(rf, 100.0, n, R, 1, MID_G, MID_A, 1, 9, lanes_per_run=lanes)
                    try:
                        res = engine.mc_free_integration(cfg, *dev)
                    except Exception as e:
                        print(json.dumps({'rf': rf, 'runs': R, 'lanes': lanes, 'shape': shape,
                                          'error': str(e)}), flush=True)
                        continue
                    torch.cuda.synchronize()
                    reps = 10 if R <= 100000 else 3
                    ms = []
                    for _ in range(reps):
                        flush.fill_(0)
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        engine.mc_free_integration(cfg, *dev, out=res)
                        e1.record()
                        torch.cuda.synchronize()
                        ms.append(e0.elapsed_time(e1))
                    m = float(np.median(ms))
                    chk = float(res.end_err.abs().sum().item())
                    print(json.dumps({'rf': rf, 'runs': R, 'n': n, 'lanes': lanes, 'shape_P_WI_split': shape,
                                      'ms': round(m, 4), 'ms_min': round(min(ms), 4),
                                      'run_steps_per_s': R * n / (m * 1e-3), 'abs_err_sum': chk}), flush=True)
    os.environ.pop('B2INS_MC_SHAPE', None)


if __name__ == '__main__':
    main()
