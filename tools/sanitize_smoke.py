"""Small invocations of every kernel family, for runs under compute-sanitizer
(memcheck / racecheck / synccheck).  GPU box only."""
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


def main():
    rng = np.random.RandomState(1)
    # K4: bulk-copy front end (4 series x 6 tiles, ragged last chunk), per-thread-load front end
    # (odd n), upper levels in one launch
    for nser, n in ((4, 30000), (3, 25001)):
        x = engine.to_device(rng.randn(nser, n) + 3.0)
        avar, tau = engine.allan(100.0, x, n, nser)
        assert torch.isfinite(avar).all()
    x = engine.to_device(rng.randn(2, 12000, 3))
    avar, _ = engine.allan(100.0, x, 12000, 6, inner=3, outer_stride=36000, sample_stride=3)
    # K4o's Hadamard form on the interleaved triads (ragged scan and output tiles)
    hvar, _ = engine.ohadamard(100.0, x, 12000, 6, inner=3, outer_stride=36000, sample_stride=3)
    assert torch.isfinite(hvar).all()
    # K13 on the transposed curves (bin stride 6, a ragged last CTA of two series)
    noise = engine.allan_fit(100.0, 12000, avar.t().contiguous(), series_stride=1, bin_stride=6)
    assert torch.isfinite(noise).all()
    # K1 (plain and time-segmented), K12 (wide and narrow groups, both frames), K3, K6
    g = {rf: dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'traj_90deg_turn_100hz_rf%d.npz' % rf)))
         for rf in (0, 1)}
    rg, ra = engine.to_device(g[1]['ref_gyro']), engine.to_device(g[1]['ref_accel'])
    engine.imu_noise(100.0, 5, rg, ra, MID_G, MID_A, 1)
    engine.imu_noise(100.0, 3, rg, ra, MID_G, MID_A, 1, layout=2)
    long_g = engine.to_device(np.zeros((300000, 3)))
    engine.imu_noise(100.0, 1, long_g, long_g, MID_G, MID_A, 1)
    for rf in (1, 0):
        gg = g[rf]
        nav = np.concatenate([gg['ref_att'], gg['ref_pos'], gg['ref_vel']], axis=1)
        dev = [engine.to_device(a) for a in (gg['ref_gyro'], gg['ref_accel'], nav, gg['ini'][None])]
        for runs, lanes in ((40, 16), (300, 1)):
            cfg = engine.make_mc_config(rf, 100.0, nav.shape[0], runs, 1, MID_G, MID_A, 1, 9, lanes_per_run=lanes)
            res = engine.mc_free_integration(cfg, *dev)
            st = engine.error_stats(res.end_err)
            assert torch.isfinite(st).all()
    # round 2: every specialised launch shape (incl. the attitude / velocity split), the fused Allan
    # experiment, the PSD FFT paths (power of two, Bluestein), the loosely-coupled filter
    gg = g[1]
    nav = np.concatenate([gg['ref_att'], gg['ref_pos'], gg['ref_vel']], axis=1)[:300]
    dev = [engine.to_device(a) for a in (gg['ref_gyro'][:300], gg['ref_accel'][:300], nav, gg['ini'][None])]
    for lanes, shape in ((1, '3,1,0'), (1, '6,1,0'), (2, '6,1,0'), (4, '3,1,1'), (4, '6,1,0'), (4, '6,2,0'), (8, '6,1,0'),
                         (8, '6,2,0'), (16, '1,4,1'), (32, '1,4,1')):
        os.environ['B2INS_MC_SHAPE'] = shape
        cfg = engine.make_mc_config(1, 100.0, 300, 37, 1, MID_G, MID_A, 1, 9, lanes_per_run=lanes, dump_runs=3)
        res = engine.mc_free_integration(cfg, *dev, dump_nav=True, dump_imu=True, dump_quat=True)
        assert torch.isfinite(res.end_err).all() and torch.isfinite(res.quat).all()
    os.environ.pop('B2INS_MC_SHAPE', None)
    z = engine.to_device(np.zeros((12000, 3)))
    avar, _ = engine.allan_mc(100.0, 3, z, z, MID_G, MID_A, 1)
    assert torch.isfinite(avar).all()
    tab = np.linspace(0, 50, 120)
    vib = {'type': 'psd', 'freq': tab, 'x': np.ones(120), 'y': np.ones(120), 'z': np.ones(120)}
    for n in (600, 20000, 9000):          # Bluestein, power of two, direct synthesis
        series, N = engine.psd_series(100.0, n, 2, 0, vib, 1)
        assert torch.isfinite(series).all()
    gp = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'gps_90deg_rf0.npz')))
    g0 = g[0]
    nav0 = np.concatenate([g0['ref_att'], g0['ref_pos'], g0['ref_vel']], axis=1)
    idx = torch.from_numpy(np.rint(gp['gps_time'] * 100.0).astype(np.int64)).cuda()
    res = engine.ins_loose(100.0, 40, 1, MID_G, MID_A, {'stdp': np.array([5.0, 5.0, 7.0]), 'stdv': np.full(3, 0.05)},
                           g0['ini'], engine.to_device(g0['ref_gyro']), engine.to_device(g0['ref_accel']),
                           engine.to_device(nav0), engine.to_device(gp['ref_gps']), idx,
                           torch.ones(len(idx), dtype=torch.float64, device='cuda'), dump_runs=2, dump_stride=10)
    assert torch.isfinite(res.end_err).all() and torch.isfinite(res.consist).all()
    # K7 with each vibration model (PSD: K5 series of exactly these 40 runs)
    n0 = g0['ref_gyro'].shape[0]
    sa, na = engine.psd_series(100.0, n0, 40, 0, vib, 1)
    sg, ng = engine.psd_series(100.0, n0, 40, 1, vib, 1)
    for vg, va in (({'type': 'random', 'x': 0.01, 'y': 0.02, 'z': 0.03}, {'type': 'random', 'x': 0.5, 'y': 0.5, 'z': 0.5}),
                   ({'type': 'sinusoidal', 'freq': 3.0, 'x': 0.01, 'y': 0.02, 'z': 0.03},
                    {'type': 'sinusoidal', 'freq': 7.5, 'x': 0.5, 'y': 0.5, 'z': 0.5}),
                   (engine.vib_series(sg * 1e-3, ng), engine.vib_series(sa, na))):
        res = engine.ins_loose(100.0, 40, 1, MID_G, MID_A, {'stdp': np.array([5.0, 5.0, 7.0]), 'stdv': np.full(3, 0.05)},
                               g0['ini'], engine.to_device(g0['ref_gyro']), engine.to_device(g0['ref_accel']),
                               engine.to_device(nav0), engine.to_device(gp['ref_gps']), idx,
                               torch.ones(len(idx), dtype=torch.float64, device='cuda'), dump_runs=2, dump_stride=10,
                               vib_gyro=vg, vib_accel=va)
        assert torch.isfinite(res.end_err).all() and torch.isfinite(res.consist).all()
    # K7's process statistics in each position frame (41 runs: a ragged last CTA), from a mid-series start
    for frame in (engine.POS_FRAME_LLA, engine.POS_FRAME_NED, engine.POS_FRAME_ECEF):
        res = engine.ins_loose(100.0, 41, 1, MID_G, MID_A, {'stdp': np.array([5.0, 5.0, 7.0]), 'stdv': np.full(3, 0.05)},
                               g0['ini'], engine.to_device(g0['ref_gyro']), engine.to_device(g0['ref_accel']),
                               engine.to_device(nav0), engine.to_device(gp['ref_gps']), idx,
                               torch.ones(len(idx), dtype=torch.float64, device='cuda'), proc_start=n0 // 3,
                               proc_pos_frame=frame)
        assert torch.isfinite(res.proc_stats).all()
    # K7 on supplied measurements (K1 / K6 output of 13 runs), with and without end_err / the initial draw
    gps_err = {'stdp': np.array([5.0, 5.0, 7.0]), 'stdv': np.full(3, 0.05)}
    fg, fa = engine.imu_noise(100.0, 13, engine.to_device(g0['ref_gyro']), engine.to_device(g0['ref_accel']),
                              MID_G, MID_A, 1)
    fgps = engine.gps_noise(13, engine.to_device(gp['ref_gps']), gps_err, 0, 1)
    vis = torch.ones(len(idx), dtype=torch.float64, device='cuda')
    for draw, nav in ((1, engine.to_device(nav0)), (0, None)):
        res = engine.ins_loose_fed(100.0, fg, fa, fgps, idx, vis, MID_G, MID_A, gps_err, g0['ini'], seed=1,
                                   ini_draw=draw, ref_nav=nav, dump_runs=2, dump_stride=10)
        assert torch.isfinite(res.end_bias).all() and torch.isfinite(res.pos).all()
    ref_gps =engine.to_device(np.tile(np.array([0.5, 2.0, 10.0, 1.0, 0.0, 0.0]), (50, 1)))
    engine.gps_noise(7, ref_gps, {'stdp': np.ones(3), 'stdv': np.ones(3)}, 0, 3)
    ref_mag = engine.to_device(np.tile(np.array([20.0, -3.0, 40.0]), (51, 1)))
    mag = engine.mag_noise(9, ref_mag, {'si': np.eye(3), 'hi': np.ones(3), 'std': np.full(3, 0.5)}, 5, 3)
    # K9 (plain, end points only, time-segmented) and K3p
    engine.imu_err_stats(100.0, 5, rg, ra, MID_G, MID_A, 1, stats_start=250)
    engine.imu_err_stats(100.0, 5, rg, ra, MID_G, MID_A, 1)
    engine.imu_err_stats(100.0, 1, long_g, long_g, MID_G, MID_A, 1, stats_start=1000)
    # K1-ex and K9-ex with the IEEE Std 952 terms: a segmented plan with a ragged last tile (n = 300 001)
    tg, ta = dict(MID_G, q=np.full(3, 1e-6), rrw=np.full(3, 2e-6), rr=np.full(3, 1e-7)), dict(MID_A, rrw=np.full(3, 1e-4))
    long_r = engine.to_device(np.zeros((300001, 3)))
    engine.imu_noise(100.0, 1, long_r, long_r, tg, ta, 1)
    engine.imu_err_stats(100.0, 1, long_r, long_r, tg, ta, 1, stats_start=1000)
    # K1-rx and K9-rx with the run-to-run errors (alone, and with the terms on the segmented plan) and their table
    xg, xa = dict(MID_G, b_std=np.full(3, 1e-5), sf=np.full(3, 1e-3), ma=1e-3), dict(MID_A, sf=np.full(3, 1e-4))
    engine.imu_noise(100.0, 5, rg, ra, xg, xa, 1)
    engine.imu_err_stats(100.0, 5, rg, ra, xg, xa, 1, stats_start=250)
    engine.imu_noise(100.0, 1, long_r, long_r, dict(tg, **xg), xa, 1)
    engine.imu_err_stats(100.0, 1, long_r, long_r, dict(tg, **xg), xa, 1, stats_start=1000)
    engine.imu_run_errors(300, xg, xa, 1, run_offset=2 ** 32 - 5)
    engine.proc_stats(mag, ref_mag, 7)
    torch.cuda.synchronize()
    print('sanitize smoke ok')


if __name__ == '__main__':
    main()
