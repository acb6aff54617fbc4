"""Where do the cycles of the warp-specialised K12 kernels go?  Uses tools/libb2ins_prof.so (built with
-DB2INS_PHASE_CLOCKS, see tools/README.md; --lib PATH loads another instrumented build).

mc_spec_kernel: per warp and per step, the cycles an integrator warp spends waiting at the hand-over
barrier / stepping, and a producer warp waiting for tiles / producing / waiting at the barrier.
mc_av_kernel (shape "6,2,0"): per warp of each role and per round of 8 samples, the attitude warp A
stepping (of which in the time-based re-evaluation after a warm block) and waiting at the round barrier, the
velocity warp V stepping and waiting, the producers waiting for tiles / producing / waiting.
Each case runs as is (idle: none) and with one role idle (B2INS_MC_DEBUG: 1 producers, 2 integrators or
A, 4 V).  `spec2_phase.py av` runs the mc_av_kernel cases only.  GPU box only."""
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import build as b  # noqa: E402
b.LIB = (sys.argv[sys.argv.index('--lib') + 1] if '--lib' in sys.argv
         else os.path.join(ROOT, 'tools', 'libb2ins_prof.so'))      # load the instrumented build
b.stale = lambda: False
from gnss_ins_sim_b200 import engine, _lib  # noqa: E402

MID_G = {'b': np.zeros(3), 'b_drift': np.full(3, 3.5 * np.pi / 180 / 3600),
         'b_corr': np.full(3, 100.0), 'arw': np.full(3, 0.25 * np.pi / 180 / 60)}
MID_A = {'b': np.zeros(3), 'b_drift': np.full(3, 5e-5), 'b_corr': np.full(3, 100.0),
         'vrw': np.full(3, 0.03 / 60)}
SPEC_CASES = [(1000, 4, '3,1,0'), (1000, 4, '3,1,1'), (1000, 4, '6,1,0'), (1000, 16, '1,4,1'), (4000, 1, '3,1,0'),
              (4000, 1, '6,1,0'), (12500, 1, '3,1,0'), (12500, 1, '6,1,0'), (12500, 2, '6,1,0'),
              (100000, 1, '6,1,0')]
AV_CASES = [(500, 8, '6,2,0'), (1000, 4, '6,2,0')]     # ref_frame 1 only
AV_ROUND = 8


def timed(diag, cfg, dev, res):
    out = (ctypes.c_ulonglong * 16)()
    diag(None, 1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    engine.mc_free_integration(cfg, *dev, out=res)
    e1.record()
    torch.cuda.synchronize()
    diag(out, 0)
    return round(e0.elapsed_time(e1), 4), out


def spec_record(rf, runs, lanes, shape, dbg, ms, out, n):
    iw = -(-runs * lanes // 32)
    pw = iw * int(shape.split(',')[0])
    return {'rf': rf, 'runs': runs, 'lanes': lanes, 'shape_P_WI_split': shape,
            'idle': {0: 'none', 1: 'producers', 2: 'integrators'}[dbg], 'ms': ms,
            'integrator_cycles_per_step': {'barrier_wait': round(out[4] / iw / n, 1),
                                           'stepping': round(out[5] / iw / n, 1)},
            'producer_cycles_per_step': {'tile_wait': round(out[0] / pw / n, 1),
                                         'producing': round(out[7] / pw / n, 1),
                                         'barrier_wait': round(out[6] / pw / n, 1)}}


def av_record(runs, lanes, dbg, ms, out, n):
    ctas = -(-runs // (32 // lanes))
    prod = 6 * (32 // lanes // 4)
    rounds = -(-n // AV_ROUND)
    per = lambda i, warps: round(out[i] / warps / rounds, 1)     # noqa: E731
    return {'rf': 1, 'runs': runs, 'lanes': lanes, 'shape_P_WI_split': '6,2,0', 'kernel': 'mc_av_kernel',
            'idle': {0: 'none', 1: 'producers', 2: 'A', 4: 'V'}[dbg], 'ms': ms,
            'A_cycles_per_round': {'stepping': per(8, ctas), 'of_which_reevaluation': per(10, ctas),
                                   'barrier_wait': per(9, ctas)},
            'V_cycles_per_round': {'stepping': per(11, ctas), 'barrier_wait': per(12, ctas)},
            'producer_cycles_per_round': {'warps_per_cta': prod, 'tile_wait': per(13, ctas * prod),
                                          'producing': per(14, ctas * prod),
                                          'barrier_wait': per(15, ctas * prod)}}


def main():
    _lib.load()
    diag = ctypes.CDLL(b.LIB).b2ins_diag_phase_clocks
    av_only = 'av' in sys.argv[1:]
    for rf in ((1,) if av_only else (1, 0)):
        g = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'traj_90deg_turn_100hz_rf%d.npz' % rf)))
        nav = np.concatenate([g['ref_att'], g['ref_pos'], g['ref_vel']], axis=1)
        n = nav.shape[0]
        dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda()
               for a in (g['ref_gyro'], g['ref_accel'], nav, g['ini'][None])]
        cases = [] if av_only else [c + (d,) for c in SPEC_CASES for d in (0, 1, 2)]
        if rf == 1:
            cases += [c + (d,) for c in AV_CASES for d in (0, 1, 2, 4)]
        for runs, lanes, shape, dbg in cases:
            os.environ['B2INS_MC_SHAPE'] = shape
            os.environ['B2INS_MC_DEBUG'] = str(dbg)
            cfg = engine.make_mc_config(rf, 100.0, n, runs, 1, MID_G, MID_A, 1, 9, lanes_per_run=lanes)
            res = engine.mc_free_integration(cfg, *dev)
            torch.cuda.synchronize()
            ms, out = timed(diag, cfg, dev, res)
            rec = (av_record(runs, lanes, dbg, ms, out, n) if shape == '6,2,0'
                   else spec_record(rf, runs, lanes, shape, dbg, ms, out, n))
            print(json.dumps(rec), flush=True)
    os.environ.pop('B2INS_MC_SHAPE', None)
    os.environ.pop('B2INS_MC_DEBUG', None)


if __name__ == '__main__':
    main()
