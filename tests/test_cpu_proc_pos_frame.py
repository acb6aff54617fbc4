"""Process-error statistics of LLA positions in NED / ECEF metres (get_error_stats('pos', err_stats_start >= 0,
extra_opt='ned' | 'ecef'), no GPU: the oracle and the host-side error of the logged-data path against the
reference's golden, and the C ABI of the option."""
import ctypes

import numpy as np
import pytest

import proc_pos_np as ppn
from conftest import load_golden

FRAMES = ['lla', 'ned', 'ecef']


def _start_idx(g, start_s):
    return int(np.where(g['time'] >= start_s)[0][0])


@pytest.mark.parametrize('frame', FRAMES)
def test_oracle_reproduces_reference_process_stats(frame):
    """The oracle applied to the frozen histories gives the reference's per-run statistics.  It takes the same
    formula (lla2ecef of both points, NED: rot_y(-pi/2 - lat) . rot_z(lon)), so only summation order differs:
    observed worst |d| 2.8e-17 m (NED), 0 (ECEF, LLA)."""
    g, s = load_golden('philox_90deg_mid_rf0.npz'), load_golden('proc_pos_stats_90deg_mid_rf0.npz')
    assert np.array_equal(s['run_ids'], g['run_ids'])
    for si, start_s in enumerate(s['starts']):
        o = ppn.process_error_stats(g['pos'], g['ref_pos'], _start_idx(g, start_s),
                                    pos_frame='' if frame == 'lla' else frame)
        for k in ('max', 'avg', 'std'):
            ref = s['proc_pos_%s_s%d_%s' % (frame, si, k)]
            assert np.abs(o[k] - ref).max() <= (1e-9 if frame != 'lla' else 1e-15), (frame, start_s, k)
    assert str(s['units_%s' % frame]) == ("['deg', 'deg', 'm']" if frame == 'lla' else "['m', 'm', 'm']")


@pytest.mark.parametrize('frame', ['ned', 'ecef'])
def test_host_lla_error_matches_oracle(frame):
    """Sim's logged-data path (host histories) converts with its own lla2ecef / ecef_to_ned rows.  Per sample the
    two differ by the rounding of two 6.4e6 m ECEF coordinates (one ulp is 9.3e-10 m): observed worst 1.1e-9 m;
    the bound is ten such ulps."""
    from gnss_ins_sim_b200.sim import lla_error_metres
    g = load_golden('philox_90deg_mid_rf0.npz')
    for r in range(g['pos'].shape[0]):
        got = lla_error_metres(g['pos'][r], g['ref_pos'], {'ned': 1, 'ecef': 2}[frame])
        ref = ppn.lla_array_error(g['pos'][r], g['ref_pos'], frame)
        assert np.abs(got - ref).max() <= 1e-8, (frame, r)


@pytest.mark.parametrize('rf,frame,ok', [(0, 3, False), (0, -1, False), (1, 1, False), (1, 2, False),
                                         (0, 1, True), (0, 2, True), (1, 0, True)])
def test_abi_checks_proc_pos_frame(rf, frame, ok):
    """The frame is checked before any device work: 0, 1 or 2, and NED / ECEF only in ref_frame 0."""
    from gnss_ins_sim_b200 import _lib, engine
    assert (_lib.POS_FRAME_LLA, _lib.POS_FRAME_NED, _lib.POS_FRAME_ECEF) == (0, 1, 2)
    err = {'b': [0.0] * 3, 'b_drift': [0.0] * 3, 'b_corr': [np.inf] * 3, 'arw': [0.0] * 3, 'vrw': [0.0] * 3}
    cfg = engine.make_mc_config(rf, 100.0, 10, 1, 1, err, err, 1, 9, stats_start=0)
    lib = _lib.load()
    rc = lib.b2ins_mc_free_integration_ex_f64(ctypes.byref(cfg), frame, *([None] * 13))
    assert rc == _lib.ERR_ARG
    msg = lib.b2ins_last_error().decode()
    if ok:     # a valid frame passes that check and fails on the missing buffers instead
        assert 'proc_pos_frame' not in msg and 'null' in msg, msg
    else:
        assert 'proc_pos_frame' in msg, msg
