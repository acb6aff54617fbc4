"""Generate tests/golden/proc_pos_stats_90deg_mid_rf0.npz by running the UNMODIFIED reference (the helpers and
the reference import of gen_golden.py).  Test infrastructure only.

    python oracle/gen_golden_proc_pos.py

get_error_stats('pos', err_stats_start, extra_opt=opt) of the reference for the philox_90deg_mid_rf0 experiment
(R = 8, seed 12345, the b2ins Philox normals injected as in gen_golden.gen_ned_stats): the per-run PROCESS
statistics (max|e|, mean, std over samples with time >= err_stats_start, ins_data_manager.py:761-795) of the
LLA position error, in LLA (opt '') or in metres (opt 'ned' / 'ecef', array_error :543-552), for
err_stats_start 0 and 2.5 s, with the output-units strings.  One fresh reference Sim per option: the
reference caches a data name's error array at its first call (:427-431).
"""
import os

import numpy as np

from gen_golden import MOTION, OUT, RandnQueue, fresh_imu, inject_stream, read_ini, ins_sim, free_integration


def gen_proc_pos_stats(R=8, seed=12345):
    csv = os.path.join(MOTION, 'motion_def-90deg_turn.csv')
    ini = read_ini(csv)
    n, run_ids = 1000, np.arange(R)
    out = {'seed': seed, 'run_ids': run_ids, 'starts': np.array([0.0, 2.5])}
    g = np.load(os.path.join(OUT, 'philox_90deg_mid_rf0.npz'))
    for opt in ('', 'ned', 'ecef'):
        sim = ins_sim.Sim([100.0, 0.0, 0.0], csv, ref_frame=0, imu=fresh_imu('mid-accuracy'),
                          algorithm=free_integration.FreeIntegration(ini))
        q = RandnQueue()
        inject_stream(q, n, run_ids, seed)
        real = np.random.randn
        np.random.randn = q
        try:
            sim.run(R)
        finally:
            np.random.randn = real
        assert not q.q
        # the runs must be the ones frozen in philox_90deg_mid_rf0.npz
        for r in range(R):
            assert np.array_equal(g['pos'][r], sim.dmgr.pos.data['algo0_%d' % r])
        tag = opt or 'lla'
        for si, start in enumerate((0, 2.5)):
            st = sim.dmgr.get_error_stats('pos', err_stats_start=start, angle=False, use_output_units=False,
                                          extra_opt=opt)
            for k in ('max', 'avg', 'std'):
                out['proc_pos_%s_s%d_%s' % (tag, si, k)] = np.stack([st[k]['algo0_%d' % r] for r in range(R)])
        st = sim.dmgr.get_error_stats('pos', err_stats_start=2.5, angle=False, use_output_units=True,
                                      extra_opt=opt)
        out['units_%s' % tag] = st['units']
    assert not np.allclose(out['proc_pos_ned_s1_std'], out['proc_pos_ecef_s1_std'])
    np.savez_compressed(os.path.join(OUT, 'proc_pos_stats_90deg_mid_rf0.npz'), **out)


if __name__ == '__main__':
    gen_proc_pos_stats()
