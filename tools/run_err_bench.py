"""What the run-to-run errors cost: K1 against K1-rx, with and without the IEEE Std 952 terms, and config 2's free
integration on K12 against K1 then K2 (the route an IMU with run errors takes).

    python tools/run_err_bench.py [--windows 5] [--runs 1000] [--n 193036]

K1 arms at --runs runs x --n samples (@100 Hz, 'mid-accuracy' IMU, a constant non-zero truth so that S ref is not
trivially zero): plain K1 against K1-rx with 'b_std', 'sf' and 'ma' on both sensors, and K1-ex (q, rrw, rr on both
sensors) against K1-ex-rx with both; CUDA events around each call.  Config 2 (motion_def-90deg_turn, n = 1000
@100 Hz, 'mid-accuracy', Sim.run(1000) with FreeIntegration + get_error_stats('pos')): K12 against K1 -> K2 with
gyro_sf = 1000 ppm, host wall clock with a device synchronise.  Window 0 warms every arm up and is not counted; the
arms alternate which goes first.  Prints the card's name and power limit (read in the same process) and one JSON
line per measurement: medians over the windows."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from gnss_ins_sim_b200 import engine, imu_model  # noqa: E402
from gnss_ins_sim_b200.sim import Sim  # noqa: E402
from gnss_ins_sim_b200.free_integration import FreeIntegration  # noqa: E402
from noise952_bench import alternate, card, events, wall  # noqa: E402

RUN_G = {'b_std': np.full(3, 5e-5), 'sf': np.full(3, 1e-3), 'ma': 1e-3}
RUN_A = {'b_std': np.full(3, 1e-2), 'sf': np.full(3, 5e-4), 'ma': 1e-3}
TERMS_G = {'q': np.full(3, 1e-6), 'rrw': np.full(3, 2e-6), 'rr': np.full(3, 1e-7)}
TERMS_A = {'q': np.full(3, 1e-4), 'rrw': np.full(3, 1e-4), 'rr': np.full(3, 1e-6)}


def imu(run=False, terms=False):
    m = imu_model.IMU('mid-accuracy', gps=False)
    m.set_gyro_error(dict(RUN_G if run else {}, **(TERMS_G if terms else {})))
    m.set_accel_error(dict(RUN_A if run else {}, **(TERMS_A if terms else {})))
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--windows', type=int, default=5)
    ap.add_argument('--runs', type=int, default=1000)
    ap.add_argument('--n', type=int, default=193036)
    args = ap.parse_args()
    print(json.dumps({'card': card()}))
    fs, R, n = 100.0, args.runs, args.n
    rg = engine.to_device(np.tile(np.array([0.01, -0.02, 0.3]), (n, 1)))
    ra = engine.to_device(np.tile(np.array([0.5, -0.3, -9.8]), (n, 1)))

    def k1(m):
        return lambda: engine.imu_noise(fs, R, rg, ra, m.gyro_err, m.accel_err, 1)

    arms = {'K1': k1(imu()), 'K1_rx': k1(imu(run=True)), 'K1_ex': k1(imu(terms=True)),
            'K1_ex_rx': k1(imu(run=True, terms=True))}
    for pair in (('K1', 'K1_rx'), ('K1_ex', 'K1_ex_rx')):
        med, raw = alternate({k: arms[k] for k in pair}, args.windows + 1, events)
        print(json.dumps({'kernels': pair, 'runs': R, 'samples': n, 'seconds_median': med,
                          'rx_over_base': med[pair[1]] / med[pair[0]],
                          'run_samples_per_s': {k: R * n / v for k, v in med.items()}, 'windows': raw}))
    del rg, ra
    torch.cuda.empty_cache()
    g = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'traj_90deg_turn_100hz_rf1.npz')))
    traj = {k: g[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    mid = imu_model.IMU('mid-accuracy', gps=False)
    sf = imu_model.IMU('mid-accuracy', gps=False)
    sf.set_gyro_error({'sf': np.full(3, 1e-3)})

    def config2(m):
        def go():
            sim = Sim([100.0, 0.0, 0.0], traj, ref_frame=1, imu=m, algorithm=FreeIntegration(g['ini']), seed=12345)
            sim.run(1000)
            sim.get_error_stats('pos', err_stats_start=-1)
        return go

    med, raw = alternate({'K12': config2(mid), 'K1_K2_sf': config2(sf)}, args.windows + 2, wall)
    print(json.dumps({'workload': 'config 2 Sim.run(1000) + get_error_stats', 'seconds_median': med,
                      'k1_k2_sf_over_k12': med['K1_K2_sf'] / med['K12'], 'windows': raw}))


if __name__ == '__main__':
    main()
