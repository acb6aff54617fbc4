"""Process-error statistics of LLA positions in NED / ECEF metres, reduced in the Monte-Carlo kernel
(b2ins_mc_config.proc_pos_frame; Sim.get_error_stats('pos', err_stats_start >= 0, extra_opt='ned' | 'ecef')),
against the reference's golden and the oracle.

Tolerance: the contract |x - ref| <= 1e-6 * max(|ref|, scale) with scale = 0.1 m, the size of the largest
position errors of these experiments (max|e| up to 0.09 m), so the floor is 1e-7 m.  What the FP64 kernel can
deliver: the error is the difference of two ECEF points of 6.4e6 m (one ulp 9.3e-10 m) converted from latitudes
that agree with the reference to a few ulps (about 1e-8 m), so agreement near 1e-8 m is expected; the floor
leaves a factor of ten."""
import os
import sys

import numpy as np
import pytest

import oracle_np as onp
import proc_pos_np as ppn
from conftest import ROOT, load_golden, assert_close

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')
REL, SCALE = 1e-6, 0.1
LANES = [1, 2, 4, 8, 16, 32]
FRAME = {'ned': 1, 'ecef': 2}
WORST = {}


@pytest.fixture(scope='module', autouse=True)
def report_worst():
    """The worst |d| [m] of each kind of comparison, printed at the end of the module (-s shows it)."""
    yield
    for k, v in sorted(WORST.items()):
        sys.stdout.write('worst |d| %-14s %.3e m\n' % (k, v))


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _errs(g):
    return ({'b': g['gyro_b'], 'b_drift': g['gyro_b_drift'], 'b_corr': g['gyro_b_corr'], 'arw': g['gyro_arw']},
            {'b': g['accel_b'], 'b_drift': g['accel_b_drift'], 'b_corr': g['accel_b_corr'], 'vrw': g['accel_vrw']})


def _traj(g):
    return {k: g[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}


def _launch(eng, g, start, frame, lanes=0, odo=False):
    ge, ae = _errs(g)
    R, n = g['gyro'].shape[:2]
    kw = {}
    if odo:
        kw = {'odo_err': {'scale': float(g['odo_scale']), 'stdv': float(g['odo_stdv'])},
              'ref_odo': _dev(g['ref_odo'])}
    cfg = eng.make_mc_config(int(g['ref_frame']), float(g['fs']), n, R, int(g['seed']), ge, ae, 1, 9,
                             run_offset=int(g['run_ids'][0]), lanes_per_run=lanes, stats_start=start,
                             proc_pos_frame=frame, **kw)
    nav = np.concatenate([g['ref_att'], g['ref_pos'], g['ref_vel']], axis=1)
    res = eng.mc_free_integration(cfg, _dev(g['ref_gyro']), _dev(g['ref_accel']), _dev(nav), _dev(g['ini'][None]))
    return res.proc_stats.cpu().numpy(), res.end_err.cpu().numpy()


def _check(got, ref, what):
    assert_close(got, ref, REL, SCALE, what)
    WORST[what.split()[0]] = max(WORST.get(what.split()[0], 0.0), float(np.abs(got - ref).max()))


@pytest.mark.parametrize('opt', ['ned', 'ecef'])
@pytest.mark.parametrize('start', [0, 250])
@pytest.mark.parametrize('lanes', LANES)
def test_kernel_proc_stats_vs_reference_and_oracle(eng, lanes, start, opt):
    g, s = load_golden('philox_90deg_mid_rf0.npz'), load_golden('proc_pos_stats_90deg_mid_rf0.npz')
    si = {0: 0, 250: 1}[start]
    assert g['time'][start] == s['starts'][si]
    ps, end = _launch(eng, g, start, FRAME[opt], lanes)
    o = ppn.process_error_stats(g['pos'], g['ref_pos'], start, pos_frame=opt)
    for k, name in enumerate(['max', 'avg', 'std']):
        _check(ps[:, k, 3:6], s['proc_pos_%s_s%d_%s' % (opt, si, name)], 'golden %s %s' % (opt, name))
        _check(ps[:, k, 3:6], o[name], 'oracle %s %s' % (opt, name))
    # attitude / velocity columns and the end-point errors are those of the LLA launch, bit for bit; the
    # LLA launch is the launch of a config that never names the frame
    lla, lla_end = _launch(eng, g, start, 0, lanes)
    ge, ae = _errs(g)
    cfg = eng.make_mc_config(0, 100.0, g['gyro'].shape[1], g['gyro'].shape[0], int(g['seed']), ge, ae, 1, 9,
                             lanes_per_run=lanes, stats_start=start)
    nav = np.concatenate([g['ref_att'], g['ref_pos'], g['ref_vel']], axis=1)
    plain = eng.mc_free_integration(cfg, _dev(g['ref_gyro']), _dev(g['ref_accel']), _dev(nav),
                                    _dev(g['ini'][None])).proc_stats.cpu().numpy()
    assert np.array_equal(lla, plain)
    assert np.array_equal(ps[:, :, 0:3], lla[:, :, 0:3]) and np.array_equal(ps[:, :, 6:9], lla[:, :, 6:9])
    assert np.array_equal(end, lla_end)
    # and the LLA launch still is the reference's LLA statistics
    for k, name in enumerate(['max', 'avg', 'std']):
        assert_close(lla[:, k, 3:6], s['proc_pos_lla_s%d_%s' % (si, name)], REL, 1e-4, 'lla ' + name)


@pytest.mark.parametrize('opt', ['ned', 'ecef'])
@pytest.mark.parametrize('tag', ['philox_90deg_mid_rf0_odo', 'philox_90deg_whitedrift_rf0'])
def test_odometer_and_white_drift_vs_oracle(eng, tag, opt):
    g = load_golden(tag + '.npz')
    for lanes in (1, 8, 32):
        ps, _ = _launch(eng, g, 250, FRAME[opt], lanes, odo=tag.endswith('_odo'))
        o = ppn.process_error_stats(g['pos'], g['ref_pos'], 250, pos_frame=opt)
        for k, name in enumerate(['max', 'avg', 'std']):
            _check(ps[:, k, 3:6], o[name], 'variants %s %s %s' % (tag, opt, name))


def _sim(rf=0, runs=8):
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    g = load_golden('philox_90deg_mid_rf%d.npz' % rf)
    imu = imu_model.IMU(accuracy='mid-accuracy', axis=6, gps=False)
    sim = Sim([100.0, 0.0, 0.0], _traj(g), ref_frame=rf, imu=imu, algorithm=FreeIntegration(g['ini']),
              seed=int(g['seed']))
    sim.run(runs)
    return sim, g


def _per_run(st, k, R=8):
    return np.stack([st[k]['algo0_%d' % r] for r in range(R)])


def test_sim_get_error_stats_and_results(eng, monkeypatch, capsys):
    sim, g = _sim()
    s = load_golden('proc_pos_stats_90deg_mid_rf0.npz')
    calls = []
    real = eng.mc_free_integration
    monkeypatch.setattr(eng, 'mc_free_integration', lambda *a, **k: (calls.append(a[0].proc_pos_frame), real(*a, **k))[1])
    sim.results(err_stats_start=2.5, extra_opt='ned')
    out = capsys.readouterr().out
    assert calls == [1], calls        # one launch for att_euler, pos and vel
    assert "statistics for simulation position from algo (in units of ['m', 'm', 'm'])" in out
    for opt in ('ned', 'ecef', ''):
        for si, start in enumerate((0.0, 2.5)):
            for units in (False, True):
                st = sim.get_error_stats('pos', start, use_output_units=units, extra_opt=opt)
                tag = opt or 'lla'
                for k in ('max', 'avg', 'std'):
                    ref = s['proc_pos_%s_s%d_%s' % (tag, si, k)]
                    if opt:
                        _check(_per_run(st, k), ref, 'sim %s %s' % (opt, k))
                    else:   # LLA: output units are deg, deg, m
                        scale = np.array([180 / np.pi, 180 / np.pi, 1.0]) if units else 1.0
                        assert_close(_per_run(st, k), ref * scale, REL, 1e-4, 'sim lla ' + k)
                if opt:
                    assert st['units'] == "['m', 'm', 'm']" == str(s['units_' + tag])
                elif units:
                    assert st['units'] == str(s['units_lla'])
    # one launch per (start, frame); the attitude and velocity columns of any of them serve
    assert sorted(calls) == [0, 0, 1, 1, 2, 2], calls
    for dn in ('att_euler', 'vel'):
        a = sim.get_error_stats(dn, 2.5, extra_opt='ned')
        b = sim.get_error_stats(dn, 2.5, extra_opt='ecef')
        c = sim.get_error_stats(dn, 2.5)
        for k in ('max', 'avg', 'std'):
            assert np.array_equal(_per_run(a, k), _per_run(b, k)) and np.array_equal(_per_run(a, k), _per_run(c, k))
    assert len(calls) == 6


def test_ref_frame_1_ignores_the_option(eng):
    sim, g = _sim(rf=1)
    for opt in ('ned', 'ecef'):
        a, b = sim.get_error_stats('pos', 2.5, extra_opt=opt), sim.get_error_stats('pos', 2.5)
        for k in ('max', 'avg', 'std'):
            assert np.array_equal(_per_run(a, k), _per_run(b, k))
        assert a['units'] == "['m', 'm', 'm']"
    o = onp.process_error_stats(g['pos'], g['ref_pos'], 250)
    assert_close(_per_run(a, 'std'), o['std'], REL, 1e-4, 'rf1 std')


def test_logged_data_directory(eng, tmp_path):
    """save_data -> a Sim on that directory: the host-history branch takes the same option."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    sim, g = _sim(runs=3)
    d = str(tmp_path / 'saved')
    sim.save_data(d, names=['time', 'ref_pos', 'ref_vel', 'ref_att_euler', 'gyro', 'accel'])
    again = Sim([100.0, 0.0, 0.0], d, ref_frame=0, imu=None, algorithm=FreeIntegration(g['ini']))
    again.run(3)
    for opt in ('ned', 'ecef'):
        a = again.get_error_stats('pos', 2.5, extra_opt=opt)
        b = sim.get_error_stats('pos', 2.5, extra_opt=opt)
        assert a['units'] == "['m', 'm', 'm']"
        o = ppn.process_error_stats(g['pos'][:3], g['ref_pos'], 250, pos_frame=opt)
        for k in ('max', 'avg', 'std'):
            _check(_per_run(a, k, 3), _per_run(b, k, 3), 'logged %s %s' % (opt, k))
            _check(_per_run(a, k, 3), o[k], 'logged-oracle %s %s' % (opt, k))
        lla = again.get_error_stats('pos', 2.5)
        assert not np.allclose(_per_run(lla, 'std', 3), _per_run(a, 'std', 3))


@pytest.mark.parametrize('rf,frame', [(0, 3), (0, -1), (1, 1), (1, 2)])
def test_abi_rejects_bad_frames(eng, rf, frame):
    g = load_golden('philox_90deg_mid_rf%d.npz' % rf)
    with pytest.raises(ValueError, match='proc_pos_frame'):
        _launch(eng, g, 0, frame)


def _worker(rank, world, port, tmp):
    import torch.distributed as td
    sys.path.insert(0, ROOT)
    torch.cuda.set_device(rank)
    td.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank,
                          world_size=world, device_id=torch.device('cuda', rank))
    from gnss_ins_sim_b200 import imu_model, dist
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    g = dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'philox_90deg_mid_rf0.npz')))
    traj = dist.broadcast_trajectory(_traj(g) if rank == 0 else None)
    imu = imu_model.IMU(accuracy='mid-accuracy', axis=6, gps=False)
    sim = Sim([100.0, 0.0, 0.0], traj, ref_frame=0, imu=imu, algorithm=FreeIntegration(g['ini']),
              seed=int(g['seed']))
    sim.run(37)                                     # uneven shards
    ps = sim.get_error_stats('pos', err_stats_start=2.5, extra_opt='ned')
    np.savez(os.path.join(tmp, 'r%d.npz' % rank), **{k: _per_run(ps, k, 37) for k in ('max', 'avg', 'std')})
    td.destroy_process_group()


def test_sharded_ned_process_stats_match_single_gpu(tmp_path):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    import torch.multiprocessing as mp
    world = 2
    port = 29700 + (os.getpid() % 1000)
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    sim, g = _sim(runs=37)
    one = sim.get_error_stats('pos', err_stats_start=2.5, extra_opt='ned')
    s = load_golden('proc_pos_stats_90deg_mid_rf0.npz')
    for r in range(world):
        z = np.load(os.path.join(str(tmp_path), 'r%d.npz' % r))
        for k in ('max', 'avg', 'std'):
            assert np.array_equal(z[k], _per_run(one, k, 37)), k
            _check(z[k][:8], s['proc_pos_ned_s1_' + k], 'sharded ' + k)

