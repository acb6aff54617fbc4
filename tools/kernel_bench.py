"""Per-kernel throughput against each kernel's own roofline (DESIGN.md section 3): achieved
algorithmic GB/s = algorithmic bytes per launch / CUDA-event time, against the measured HBM
copy bandwidth (MEASURED_PEAKS.json), and run-steps/s against the measured FP64-FMA issue rate
for the FP64-bound kernels.  One JSON line per measurement.  GPU box only."""
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gnss_ins_sim_b200 import engine, _lib  # noqa: E402

MID_G = {'b': np.zeros(3), 'b_drift': np.full(3, 3.5 * np.pi / 180 / 3600),
         'b_corr': np.full(3, 100.0), 'arw': np.full(3, 0.25 * np.pi / 180 / 60)}
MID_A = {'b': np.zeros(3), 'b_drift': np.full(3, 5e-5), 'b_corr': np.full(3, 100.0),
         'vrw': np.full(3, 0.03 / 60)}


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    ms = []
    for _ in range(reps):
        flush.fill_(0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def emit(**kw):
    print(json.dumps(kw), flush=True)


def main():
    only = sys.argv[1] if len(sys.argv) > 1 else ''
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))
    except OSError:
        pass
    hbm = float(peaks.get('hbm_gbs', 3350.0))     # fallback: H100 SXM data sheet
    dfma = ctypes.c_double()
    _lib.check(_lib.load().b2ins_diag_dfma_rate(ctypes.byref(dfma)))
    emit(kernel='peaks', hbm_gbs=hbm, hbm_source='MEASURED_PEAKS.json' if peaks else 'fallback',
         dfma_per_s=dfma.value)
    g = {rf: dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'traj_90deg_turn_100hz_rf%d.npz' % rf)))
         for rf in (0, 1)}

    # ---- K12 fused Monte-Carlo ---------------------------------------------------------
    for rf in ((1, 0) if only in ('', 'K12') else ()):
        gg = g[rf]
        nav = np.concatenate([gg['ref_att'], gg['ref_pos'], gg['ref_vel']], axis=1)
        n = nav.shape[0]
        dev = [engine.to_device(a) for a in (gg['ref_gyro'], gg['ref_accel'], nav, gg['ini'][None])]
        for runs in (1000, 10000, 100000, 1000000):
            cfg = engine.make_mc_config(rf, 100.0, n, runs, 1, MID_G, MID_A, 1, 9)
            res = engine.mc_free_integration(cfg, *dev)
            ms = timed(lambda: engine.mc_free_integration(cfg, *dev, out=res), reps=5 if runs < 1e6 else 3)
            rate = runs * n / (ms * 1e-3)
            alg = n * 48 + 144 + runs * 72
            emit(kernel='K12 mc_kernel fused', ref_frame=rf, runs=runs, n=n, ms=ms, run_steps_per_s=rate,
                 dfma_slots_per_run_step=dfma.value / rate, alg_bytes=alg,
                 alg_gbs=alg / ms / 1e6, hbm_frac=alg / ms / 1e6 / hbm)

    # ---- K2 fed-noise (120 B per run-step: 48 read + 72 written) -------------------------
    gg = g[1]
    for layout, runs, n, lanes in (((0, 4096, 1000, 0), (0, 32768, 500, 8), (1, 65536, 500, 1),
                                    (1, 262144, 250, 1)) if only in ('', 'K2') else ()):
        shape = (runs, n, 3) if layout == 0 else (n, 3, runs)
        gyro = torch.randn(shape, dtype=torch.float64, device='cuda') * 0.01
        accel = torch.randn(shape, dtype=torch.float64, device='cuda') * 0.1
        accel[..., 2] -= 9.8 if layout == 0 else 0.0
        ini = engine.to_device(gg['ini'][None])
        ms = timed(lambda: engine.free_integration(1, 100.0, gyro, accel, ini, layout=layout,
                                                   lanes_per_run=lanes), reps=3)
        rate = runs * n / (ms * 1e-3)
        emit(kernel='K2 mc_kernel fed', layout='run-major' if layout == 0 else 'time-major', runs=runs,
             n=n, lanes=lanes or 'auto', ms=ms, run_steps_per_s=rate, alg_gbs=rate * 120 / 1e9,
             hbm_frac=rate * 120 / 1e9 / hbm, dfma_slots_per_run_step=dfma.value / rate)
        del gyro, accel

    # ---- K1 materialised noise (48 B written per run-step) --------------------------------
    rg = torch.zeros((4000, 3), dtype=torch.float64, device='cuda')
    for runs in ((1024, 8192, 65536) if only in ('', 'K1') else ()):
        ms = timed(lambda: engine.imu_noise(100.0, runs, rg, rg, MID_G, MID_A, 1), reps=3)
        rate = runs * 4000 / (ms * 1e-3)
        emit(kernel='K1 imu_noise_kernel', runs=runs, n=4000, ms=ms, run_steps_per_s=rate,
             alg_gbs=rate * 48 / 1e9, hbm_frac=rate * 48 / 1e9 / hbm,
             dfma_slots_per_run_step=dfma.value / rate)

    # ---- K3 statistics (72 B per run read twice) -------------------------------------------
    for runs in ((1000, 1000000) if only in ('', 'K3') else ()):
        err = torch.randn((runs, 9), dtype=torch.float64, device='cuda')
        ms = timed(lambda: engine.error_stats(err), reps=5)
        emit(kernel='K3 error_stats', runs=runs, ms=ms, alg_gbs=runs * 72 * 2 / ms / 1e6,
             hbm_frac=runs * 72 * 2 / ms / 1e6 / hbm)

    # ---- K4 Allan (8 B per sample read once + 0.8 B decade sums) ---------------------------
    for nser, n, inner in (((96, 2000000, 1), (32, 2000000, 3), (6, 14400000, 3)) if only in ('', 'K4') else ()):
        x = torch.randn(nser * n, dtype=torch.float64, device='cuda')
        if inner == 1:
            fn = lambda: engine.allan(400.0, x, n, nser)                                   # noqa: E731
        else:
            fn = lambda: engine.allan(400.0, x, n, nser, inner=3, outer_stride=3 * n, sample_stride=3)  # noqa: E731
        ms = timed(fn, reps=3)
        emit(kernel='K4 allan', series=nser, n=n, interleave=inner, ms=ms,
             samples_per_s=nser * n / (ms * 1e-3), alg_gbs=nser * n * 8.8 / ms / 1e6,
             hbm_frac=nser * n * 8.8 / ms / 1e6 / hbm)
        del x

    # ---- K14 Allan with the series generated in the tile (K1 fused into K4) -----------------
    for runs, n in (((64, 2000000), (256, 14400000)) if only in ('', 'K14') else ()):
        rz = torch.zeros((n, 3), dtype=torch.float64, device='cuda')
        ms = timed(lambda: engine.allan_mc(400.0, runs, rz, rz, MID_G, MID_A, 1), reps=2, warm=1)
        emit(kernel='K14 allan_gen (fused K1+K4)', runs=runs, n=n, ms=ms,
             sample_channels_per_s=runs * 6 * n / (ms * 1e-3),
             dfma_slots_per_sample_channel=dfma.value / (runs * 6 * n / (ms * 1e-3)))
        del rz

    # ---- K7 loosely-coupled filter -----------------------------------------------------------
    if only in ('', 'K7'):
        gg0 = g[0]
        gp = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'gps_90deg_rf0.npz')))
        nav0 = np.concatenate([gg0['ref_att'], gg0['ref_pos'], gg0['ref_vel']], axis=1)
        d0 = [engine.to_device(a) for a in (gg0['ref_gyro'], gg0['ref_accel'], nav0, gp['ref_gps'])]
        idx = torch.from_numpy(np.rint(gp['gps_time'] * 100.0).astype(np.int64)).cuda()
        vis = torch.ones(len(idx), dtype=torch.float64, device='cuda')
        gerr = {'stdp': np.array([5.0, 5.0, 7.0]), 'stdv': np.array([0.05, 0.05, 0.05])}
        for runs in (1250, 10000, 100000):
            ms = timed(lambda: engine.ins_loose(100.0, runs, 1, MID_G, MID_A, gerr, gg0['ini'], d0[0], d0[1], d0[2],
                                                d0[3], idx, vis), reps=3)
            emit(kernel='K7 ekf_kernel', runs=runs, n=1000, ms=ms, run_steps_per_s=runs * 1000 / (ms * 1e-3))

    # ---- K5 PSD series ----------------------------------------------------------------------
    tab = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'psd.npz')))
    vib = {'type': 'psd', 'freq': tab['freq_a'], 'x': tab['sxx_a'], 'y': tab['sxx_a'], 'z': tab['sxx_a']}
    for runs, n in (((64, 1000), (64, 40000), (2048, 1000), (2048, 6000), (2048, 40000)) if only in ('', 'K5') else ()):
        ms = timed(lambda: engine.psd_series(200.0, n, runs, 0, vib, 1), reps=3)
        emit(kernel='K5 psd_series', runs=runs, n=n, ms=ms, series_per_s=runs * 3 / (ms * 1e-3))


if __name__ == '__main__':
    main()
