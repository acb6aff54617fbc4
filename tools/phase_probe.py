"""Where do the cycles of mc_kernel go?  Uses tools/libb2ins_prof.so (built with
-DB2INS_PHASE_CLOCKS): cumulative warp-cycles in tile wait / phase A (noise) / phase A + GM
scan / phase B per (runs, lanes, ref_frame).  GPU box only."""
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import build as b  # noqa: E402
b.LIB = os.path.join(ROOT, 'tools', 'libb2ins_prof.so')      # load the instrumented build
b.stale = lambda: False
from gnss_ins_sim_b200 import engine, _lib  # noqa: E402


def main():
    _lib.load()
    diag = ctypes.CDLL(b.LIB).b2ins_diag_phase_clocks
    mid_g = {'b': np.zeros(3), 'b_drift': np.full(3, 3.5 * np.pi / 180 / 3600),
             'b_corr': np.full(3, 100.0), 'arw': np.full(3, 0.25 * np.pi / 180 / 60)}
    mid_a = {'b': np.zeros(3), 'b_drift': np.full(3, 5e-5), 'b_corr': np.full(3, 100.0),
             'vrw': np.full(3, 0.03 / 60)}
    for rf in (1, 0):
        g = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'traj_90deg_turn_100hz_rf%d.npz' % rf)))
        nav = np.concatenate([g['ref_att'], g['ref_pos'], g['ref_vel']], axis=1)
        n = nav.shape[0]
        dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda()
               for a in (g['ref_gyro'], g['ref_accel'], nav, g['ini'][None])]
        for runs, lanes in ((1000, 8), (1000, 16), (1000, 32), (100000, 1), (1000000, 1)):
            cfg = engine.make_mc_config(rf, 100.0, n, runs, 1, mid_g, mid_a, 1, 9, lanes_per_run=lanes)
            res = engine.mc_free_integration(cfg, *dev)
            torch.cuda.synchronize()
            out = (ctypes.c_ulonglong * 16)()
            diag(None, 1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            engine.mc_free_integration(cfg, *dev, out=res)
            e1.record()
            torch.cuda.synchronize()
            diag(out, 0)
            warps = -(-runs * lanes // 32)
            c = [out[i] / warps / n for i in range(4)]
            print(json.dumps({'rf': rf, 'runs': runs, 'lanes': lanes, 'ms': round(e0.elapsed_time(e1), 4),
                              'cycles_per_step_per_warp': {'tile_wait': round(c[0], 1),
                                                           'phaseA_noise': round(c[1], 1),
                                                           'gm_scan': round(c[2] - c[1], 1),
                                                           'phaseB': round(c[3], 1)}}), flush=True)


if __name__ == '__main__':
    main()
