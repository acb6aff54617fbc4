"""Per-run process-error statistics of the loosely-coupled filter (K7's PROC form): b2ins_ins_loose_proc_f64,
engine.ins_loose(proc_start=...) and Sim.get_error_stats / results() with err_stats_start >= 0.

The statistics are held to the spec (oracle/ekf_proc_np.py) on identical draws, to the host statistics of the
same launch's histories, and leave every other output of the filter unchanged; through Sim they are one
launch per (start, frame), in run blocks with PSD vibration."""
import numpy as np
import pytest

from conftest import load_golden, assert_close
import ekf_proc_np
from proc_pos_np import lla_array_error

torch = pytest.importorskip('torch')
gpu = pytest.mark.gpu
FS = 100.0
DEMO_IMU = {'gyro_b': np.zeros(3), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
            'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
            'accel_b': np.zeros(3), 'accel_vrw': np.array([0.03119, 0.03009, 0.04779]),
            'accel_b_stability': np.array([4.29e-5, 5.72e-5, 8.02e-5]),
            'accel_b_corr': np.array([200.0, 200.0, 200.0])}       # demo_ins_loose.py:28-37
PSD = np.stack([np.linspace(0.0, 50.0, 26), np.full(26, 1e-2), np.linspace(1e-2, 4e-2, 26),
                np.full(26, 2e-2)], axis=1)
R, R0, SEED = 13, 5, 2025        # two CTAs of eight runs, the second ragged, from run 5


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _imu():
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True)


def _turn_case():
    """The 90-degree-turn trajectory in ref_frame 0 with its 10 Hz GPS truth, all GPS samples visible."""
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    g = dict(load_golden('gps_90deg_rf0.npz'))
    g['gps_visibility'] = np.ones_like(g['gps_visibility'])
    nav = np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1)
    idx = np.rint(g['gps_time'] * 100.0).astype(np.int64)
    return t, g, nav, idx


def _launch(eng, t, g, nav, idx, imu, runs, **kw):
    dev = [eng.to_device(a) for a in (t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'])]
    return eng.ins_loose(FS, runs, SEED, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'], dev[0], dev[1],
                         dev[2], dev[3], torch.from_numpy(idx).cuda(),
                         eng.to_device(np.asarray(g['gps_visibility'], dtype=np.float64)), **kw)


def _spec(t, g, nav, idx, imu, start, **kw):
    return ekf_proc_np.ins_loose(FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                                 imu.gyro_err, imu.accel_err, imu.gps_err, SEED, np.arange(R0, R0 + R), t['ini'],
                                 start, **kw)


def _assert_stats(ps, ref, nav, frame, what):
    """The tolerances test_ekf.test_kernel_equals_the_spec holds K7's histories to, carried to max|e|, mean
    and std (each moves by at most the largest per-sample difference): attitude 1e-9 rad; lat / lon / alt
    1e-9 of the truth's magnitude (in NED / ECEF metres, 1e-9 of an Earth radius); velocity 1e-9 of the
    truth's magnitude."""
    assert_close(ps[:, :, 0:3], ref[:, :, 0:3], 1e-9, 1.0, what + ' att')
    if frame == '':
        scale = np.maximum(np.abs(nav[:, 3:6]).max(0), [1e-4, 1e-4, 1e-2])
        assert_close(ps[:, :, 3:6], ref[:, :, 3:6], 1e-9, scale, what + ' lat/lon/alt')
    else:
        assert_close(ps[:, :, 3:6], ref[:, :, 3:6], 1e-9, 6.4e6, what + ' pos m')
    assert_close(ps[:, :, 6:9], ref[:, :, 6:9], 1e-9, np.maximum(np.abs(nav[:, 6:9]).max(0), 1e-2), what + ' vel')
    print(what, 'worst |kernel - spec| (att, pos, vel):',
          [float(np.abs(ps[:, :, c:c + 3] - ref[:, :, c:c + 3]).max()) for c in (0, 3, 6)])


@gpu
def test_kernel_equals_the_spec(eng):
    """13 runs from run 5, every frame, starts 0, mid-series and the last sample."""
    t, g, nav, idx = _turn_case()
    imu = _imu()
    n = t['ref_gyro'].shape[0]
    h = _spec(t, g, nav, idx, imu, 0, stats_start=100)
    for fi, frame in enumerate(ekf_proc_np.FRAMES):
        for start in (0, n // 2 + 3, n - 1):
            ref = ekf_proc_np.process_stats(h['att'], h['pos'], h['vel'], nav, start, frame)
            res = _launch(eng, t, g, nav, idx, imu, R, run_offset=R0, stats_start=100, vel_rw=0.0,
                          proc_start=start, proc_pos_frame=fi)
            ps = res.proc_stats.cpu().numpy()
            assert ps.shape == (R, 3, 9)
            _assert_stats(ps, ref, nav, frame, '%r start %d' % (frame, start))
            if start == n - 1:
                assert np.all(ps[:, 2] == 0.0)


@gpu
def test_statistics_of_the_launch_own_histories(eng):
    """Row i after its GPS update, the last sample included: the statistics equal NumPy's over the histories
    the same launch dumps, in LLA (the same error values on both sides: only the summation differs)."""
    t, g, nav, idx = _turn_case()
    imu = _imu()
    start = 777
    res = _launch(eng, t, g, nav, idx, imu, R, run_offset=R0, proc_start=start, dump_runs=R)
    ps = res.proc_stats.cpu().numpy()
    host = ekf_proc_np.process_stats(res.att.cpu().numpy(), res.pos.cpu().numpy(), res.vel.cpu().numpy(), nav,
                                     start, '')
    scale = np.abs(host).max(axis=0, keepdims=True)        # per statistic and column, over the runs
    assert np.all(np.abs(ps - host) <= 1e-12 * scale), np.abs(ps - host).max()
    # metres: the same rows through lla2ecef on the host
    res_ned = _launch(eng, t, g, nav, idx, imu, R, run_offset=R0, proc_start=start, proc_pos_frame=1)
    e = lla_array_error(res.pos.cpu().numpy()[:, start:], nav[None, start:, 3:6], 'ned')
    assert_close(res_ned.proc_stats.cpu().numpy()[:, 1, 3:6], e.mean(1), 1e-9, 1e2, 'NED mean of own rows')


@gpu
def test_statistics_leave_the_filter_unchanged(eng):
    t, g, nav, idx = _turn_case()
    imu = _imu()
    keys = ('end_err', 'end_bias', 'consist', 'att', 'pos', 'vel', 'wb', 'ab')
    plain = _launch(eng, t, g, nav, idx, imu, R, run_offset=R0, stats_start=100, dump_runs=R, dump_stride=3)
    for frame in (0, 1, 2):
        proc = _launch(eng, t, g, nav, idx, imu, R, run_offset=R0, stats_start=100, dump_runs=R, dump_stride=3,
                       proc_start=50, proc_pos_frame=frame)
        for k in keys:
            assert np.array_equal(getattr(proc, k).cpu().numpy(), getattr(plain, k).cpu().numpy()), (frame, k)
    assert plain.proc_stats is None


@gpu
def test_vibrating_kernel_equals_the_spec(eng):
    """ekf_kernel<true, false, true>: random vibration on both sensors."""
    from gnss_ins_sim_b200.sim import parse_env
    t, g, nav, idx = _turn_case()
    imu = _imu()
    va, vg = parse_env('[0.05 0.05 0.05]g-random', FS), parse_env('[0.5 0.5 0.5]d-random', FS)
    start = 401
    h = _spec(t, g, nav, idx, imu, start, stats_start=100, vib_acc=va, vib_gyro=vg)
    for fi, frame in ((0, ''), (1, 'ned')):
        ref = ekf_proc_np.process_stats(h['att'], h['pos'], h['vel'], nav, start, frame)
        res = _launch(eng, t, g, nav, idx, imu, R, run_offset=R0, stats_start=100, vel_rw=0.0, vib_accel=va,
                      vib_gyro=vg, proc_start=start, proc_pos_frame=fi)
        _assert_stats(res.proc_stats.cpu().numpy(), ref, nav, frame, 'vibration %r' % frame)


# ---- through Sim ----------------------------------------------------------------------------------------
def _sim(env=None):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.ins_loose import InsLoose
    gm = load_golden('philox_90deg_mid_rf0.npz')
    gp = load_golden('gps_90deg_rf0.npz')
    traj = {k: gm[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro', 'ini')}
    traj.update(ref_gps=gp['ref_gps'], gps_time=gp['gps_time'], gps_visibility=np.ones_like(gp['gps_visibility']))
    return Sim([FS, 10.0, 0.0], traj, ref_frame=0, imu=_imu(), env=env, algorithm=InsLoose(gm['ini']), seed=5,
               history_block=8)


def _count(monkeypatch, eng):
    calls = []
    real = eng.ins_loose
    monkeypatch.setattr(eng, 'ins_loose', lambda *a, **k: calls.append((a[1], k.get('run_offset'),
                                                                        k.get('proc_start'),
                                                                        k.get('proc_pos_frame'))) or real(*a, **k))
    return calls


@gpu
def test_sim_psd_run_blocks_equal_one_block(eng, monkeypatch):
    env = {'acc': PSD, 'gyro': PSD * 1e-4}
    one, blocks = _sim(env), _sim(env)
    one.run(20)
    blocks.run(20)
    monkeypatch.setattr(blocks, '_allan_block', lambda *a: 6)
    calls = _count(monkeypatch, eng)
    a = one.get_error_stats('pos', err_stats_start=2.0, extra_opt='ned')
    b = blocks.get_error_stats('pos', err_stats_start=2.0, extra_opt='ned')
    assert [c[:2] for c in calls] == [(20, 0), (6, 0), (6, 6), (6, 12), (2, 18)]
    for k in ('max', 'avg', 'std'):
        assert sorted(a[k]) == sorted(b[k]) and len(a[k]) == 20
        for r in a[k]:
            assert np.array_equal(a[k][r], b[k][r]), (k, r)


@gpu
def test_sim_error_stats_and_results(eng, monkeypatch, capsys):
    sim = _sim()
    sim.run(11)
    calls = _count(monkeypatch, eng)
    names = sim.results()                   # err_stats_start = 0: per-run process statistics
    assert names and 'Simulation run algo0_10' in capsys.readouterr().out
    assert calls == [(11, 0, 0, 0)]
    # the statistics are the engine's on the same runs, from the first sample at or after 3 s
    d = sim._dev
    start = int(np.searchsorted(sim.data['time'], 3.0))
    for fi, opt in enumerate(('', 'ned', 'ecef')):
        st = sim.get_error_stats('pos', err_stats_start=3.0, extra_opt=opt)
        assert st['units'] == ("['m', 'm', 'm']" if opt else "['rad', 'rad', 'm']")
        direct = eng.ins_loose(FS, 11, 5, sim.imu.gyro_err, sim.imu.accel_err, sim.imu.gps_err, sim.algo[0].ini,
                               d['ref_gyro'], d['ref_accel'], d['ref_nav'], d['ref_gps'], d['gps_idx'],
                               d['gps_vis'], vel_rw=sim.algo[0].vel_model_std, att_rw=sim.algo[0].att_model_std,
                               proc_start=start, proc_pos_frame=fi).proc_stats.cpu().numpy()
        for k, s in enumerate(('max', 'avg', 'std')):
            for r in (0, 7, 10):
                assert np.array_equal(st[s]['algo0_%d' % r], direct[r, k, 3:6]), (opt, s, r)
    launched = len(calls)
    assert [c[2:] for c in calls[1:launched:2]] == [(start, 0), (start, 1), (start, 2)]
    att = sim.get_error_stats('att_euler', err_stats_start=3.0, use_output_units=True)
    vel = sim.get_error_stats('vel', err_stats_start=3.0)
    sim.get_error_stats('pos', err_stats_start=3.0, extra_opt='ned')
    assert len(calls) == launched           # repeated and cross-frame calls launch nothing
    assert att['units'] == "['deg', 'deg', 'deg']" and vel['units'] == "['m/s', 'm/s', 'm/s']"
    assert len(att['max']) == 11 and np.all(np.isfinite(att['std']['algo0_3']))


@gpu
def test_argument_errors(eng, monkeypatch):
    t, g, nav, idx = _turn_case()
    imu = _imu()
    n = t['ref_gyro'].shape[0]
    for start in (-1, n):
        with pytest.raises(ValueError, match=r'proc_start must be in \[0, n\)'):
            _launch(eng, t, g, nav, idx, imu, 4, proc_start=start)
    with pytest.raises(ValueError, match='proc_pos_frame must be B2INS_POS_FRAME_'):
        _launch(eng, t, g, nav, idx, imu, 4, proc_start=0, proc_pos_frame=3)
    lib = eng._lib.load()
    real = lib.b2ins_ins_loose_proc_f64

    class NoStats(object):      # the library with proc_stats dropped from the call
        def __getattr__(self, name):
            return getattr(lib, name)

        @staticmethod
        def b2ins_ins_loose_proc_f64(*a):
            a = list(a)
            a[14] = None
            return real(*a)
    monkeypatch.setattr(eng._lib, 'load', lambda: NoStats())
    with pytest.raises(ValueError, match='proc_stats is required'):
        _launch(eng, t, g, nav, idx, imu, 4, proc_start=0)
