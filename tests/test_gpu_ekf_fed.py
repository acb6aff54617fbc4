"""The loosely-coupled filter (K7) on supplied measurements: ekf_kernel<false, true> through
b2ins_ins_loose_fed_f64, engine.ins_loose_fed, InsLoose.run_batch / run and Sim on a logged-data directory.

The kernel is held to the fed spec (oracle/ekf_fed_np.py) on data the generator never makes; fed the generator's
own measurements (K1, K6) with the same initial draw it reproduces the generated experiment; a generated
experiment saved with save_data filters back to itself; and the plugin works in the reference's per-run
protocol."""
import copy

import numpy as np
import pytest

from conftest import load_golden, assert_close, wrap_pi
import ekf_fed_np
import oracle_np as onp

torch = pytest.importorskip('torch')
gpu = pytest.mark.gpu
FS = 100.0
DEMO_IMU = {'gyro_b': np.zeros(3), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
            'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
            'accel_b': np.zeros(3), 'accel_vrw': np.array([0.03119, 0.03009, 0.04779]),
            'accel_b_stability': np.array([4.29e-5, 5.72e-5, 8.02e-5]),
            'accel_b_corr': np.array([200.0, 200.0, 200.0])}       # demo_ins_loose.py:28-37


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _imu():
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True)


def _turn():
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    g = load_golden('gps_90deg_rf0.npz')
    nav = np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1)
    return t, g, nav


def _close(got, ref, what=''):
    """The tolerances of test_ekf.py::test_kernel_equals_the_spec.  got / ref: dicts of att, pos, vel, wb, ab
    histories and (optionally) end_err, end_bias; returns the largest absolute difference of each."""
    assert np.abs(wrap_pi(got['att'] - ref['att'])).max() < 1e-9, what
    assert_close(got['pos'][..., :2], ref['pos'][..., :2], 1e-9, 1e-4, what + ' lat/lon')
    assert_close(got['pos'][..., 2], ref['pos'][..., 2], 1e-9, 1e-2, what + ' alt')
    assert_close(got['vel'], ref['vel'], 1e-9, 1e-2, what + ' vel')
    assert_close(got['wb'], ref['wb'], 1e-7, 1e-6, what + ' gyro bias estimate')
    assert_close(got['ab'], ref['ab'], 1e-7, 1e-5, what + ' accel bias estimate')
    for k in ('end_err', 'end_bias'):
        if k in ref:
            assert_close(got[k], ref[k], 1e-7, 1e-6, what + ' ' + k)
    return {k: float(np.abs(wrap_pi(got[k] - ref[k]) if k == 'att' else got[k] - ref[k]).max())
            for k in ref if k in got}


def _host(res):
    out = {'att': res.att, 'pos': res.pos, 'vel': res.vel, 'wb': res.wb, 'ab': res.ab, 'end_bias': res.end_bias}
    if res.end_err is not None:
        out['end_err'] = res.end_err
    return {k: v.cpu().numpy() for k, v in out.items()}


@gpu
@pytest.mark.parametrize('ini_draw', [0, 1])
def test_kernel_equals_the_fed_spec(eng, ini_draw):
    """The 90-degree turn with measurements the generator never makes: another seed's IMU noise, GPS thinned to
    5 Hz from 0.3 s on (the first update is not at sample 0), a visibility-0 outage; 13 runs (a ragged last CTA)."""
    t, g, nav = _turn()
    imu = _imu()
    R, r0, seed = 13, 21, 909
    run_ids = np.arange(R) + 500
    gyro, accel = onp.imu_noise(FS, t['ref_gyro'], t['ref_accel'], imu.gyro_err, imu.accel_err, 31, run_ids)
    rows = np.arange(3, g['ref_gps'].shape[0], 2)
    gps = onp.gps_gen(g['ref_gps'], imu.gps_err, 0, onp.gps_normals(g['ref_gps'].shape[0], run_ids, 31))[:, rows]
    idx = np.rint(g['gps_time'][rows] * FS).astype(np.int64)
    vis = np.ones(rows.size)
    vis[10:16] = 0.0
    o = ekf_fed_np.ins_loose(FS, gyro, accel, gps, idx, vis, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'],
                             seed=seed, run_ids=np.arange(r0, r0 + R), ini_draw=bool(ini_draw), ref_nav=nav,
                             want_hist=True, vel_rw=0.02)
    dev = [eng.to_device(a) for a in (gyro, accel, gps)]
    args = (FS, *dev, torch.from_numpy(idx).cuda(), eng.to_device(vis), imu.gyro_err, imu.accel_err, imu.gps_err,
            t['ini'])
    res = eng.ins_loose_fed(*args, seed=seed, ini_draw=ini_draw, run_offset=r0, ref_nav=eng.to_device(nav),
                            dump_runs=R)
    assert res.consist is None
    _close(_host(res), o, 'ini_draw=%d' % ini_draw)
    if not ini_draw:      # every run starts at ini (through the DCM round trip of the attitude)
        assert np.array_equal(res.pos[:, 0].cpu().numpy(), np.tile(t['ini'][0:3], (R, 1)))
    # decimated histories are rows of the full ones; without ref_nav there is no end_err and the rest is the same
    dec = eng.ins_loose_fed(*args, seed=seed, ini_draw=ini_draw, run_offset=r0, dump_runs=5, dump_stride=7)
    assert dec.end_err is None
    assert np.array_equal(dec.pos.cpu().numpy(), res.pos[:5, ::7].cpu().numpy())
    assert np.array_equal(dec.end_bias.cpu().numpy(), res.end_bias.cpu().numpy())


def _generated_vs_fed(eng, vib_acc=None, vib_gyro=None):
    t, g, nav = _turn()
    imu = _imu()
    R, r0, seed = 21, 7, 4711
    gps_t = dict(g)
    idx = np.rint(g['gps_time'] * FS).astype(np.int64)
    vis = np.ones(idx.size)
    vis[30:40] = 0.0
    ref = [eng.to_device(a) for a in (t['ref_gyro'], t['ref_accel'], nav, gps_t['ref_gps'])]
    d_idx, d_vis = torch.from_numpy(idx).cuda(), eng.to_device(vis)
    gen = eng.ins_loose(FS, R, seed, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'], *ref, d_idx, d_vis,
                        run_offset=r0, dump_runs=R, vib_gyro=vib_gyro, vib_accel=vib_acc)
    gyro, accel = eng.imu_noise(FS, R, ref[0], ref[1], imu.gyro_err, imu.accel_err, seed, run_offset=r0,
                                vib_gyro=vib_gyro, vib_accel=vib_acc)
    gps = eng.gps_noise(R, ref[3], imu.gps_err, 0, seed, run_offset=r0)
    fed = eng.ins_loose_fed(FS, gyro, accel, gps, d_idx, d_vis, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'],
                            seed=seed, ini_draw=True, run_offset=r0, ref_nav=ref[2], dump_runs=R)
    return _close(_host(fed), _host(gen), 'fed vs generated')


@gpu
def test_fed_equals_generated(eng):
    """K1's and K6's measurements of the same runs, with the same initial draw, filter to the generated
    experiment: the same filter on the same numbers up to K1's association of the Gauss-Markov scan."""
    print('largest |fed - generated|:', _generated_vs_fed(eng))


@gpu
def test_fed_equals_generated_with_random_vibration(eng):
    from gnss_ins_sim_b200.sim import parse_env
    d = _generated_vs_fed(eng, parse_env('[0.05 0.05 0.05]g-random', FS), parse_env('[0.5 0.5 0.5]d-random', FS))
    print('largest |fed - generated| with random vibration:', d)


# ---- through Sim and the plugin ----------------------------------------------------------------------------
def _traj():
    gm = load_golden('philox_90deg_mid_rf0.npz')
    gp = load_golden('gps_90deg_rf0.npz')
    traj = {k: gm[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro', 'ini')}
    traj.update(ref_gps=gp['ref_gps'], gps_time=gp['gps_time'], gps_visibility=np.ones_like(gp['gps_visibility']))
    traj['gps_visibility'][40:52] = 0.0
    return traj


@gpu
def test_saved_experiment_filters_back_to_itself(eng, tmp_path):
    """A generated filter experiment written with save_data and read back as a logged-data directory: the same
    histories, bias estimates and end-point statistics, up to the ulps of the text files and deg <-> rad."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.ins_loose import InsLoose
    traj, imu, R = _traj(), _imu(), 11
    gen = Sim([FS, 10.0, 0.0], traj, ref_frame=0, imu=imu, algorithm=InsLoose(traj['ini'], imu=imu), seed=5,
              run_base=3)
    gen.run(R)
    gen.save_data(str(tmp_path), names=['time', 'gyro', 'accel', 'gps', 'gps_time', 'gps_visibility', 'ref_pos',
                                        'ref_vel', 'ref_att_euler'])
    assert not list(tmp_path.glob('pos-*'))
    fed = Sim([FS, 10.0, 0.0], str(tmp_path), ref_frame=0, algorithm=InsLoose(traj['ini'], imu=imu), seed=5,
              run_base=3)
    fed.run(R)
    names = ['att_euler', 'pos', 'vel', 'wb', 'ab']
    a, b = gen.get_data(names), fed.get_data(names)
    for r in range(R):
        key = 'algo0_%d' % r
        _close({k: b[i][key] for i, k in enumerate(('att', 'pos', 'vel', 'wb', 'ab'))},
               {k: a[i][key] for i, k in enumerate(('att', 'pos', 'vel', 'wb', 'ab'))}, key)
    assert_close(fed.end_point_errors(), gen.end_point_errors(), 1e-7, 1e-6, 'end-point errors')
    assert_close(fed._mc[0]['end_bias'], gen._mc[0]['end_bias'], 1e-7, 1e-6, 'end biases')
    for name in ('pos', 'vel', 'att_euler'):
        sg, sf = gen.get_error_stats(name, -1), fed.get_error_stats(name, -1)
        for k in ('max', 'avg', 'std'):
            assert_close(sf[k], sg[k], 1e-6, 1e-9 if name != 'vel' else 1e-6, '%s %s' % (name, k))
    st = fed.get_error_stats('pos', 2.0)          # per-run process statistics through the logged path
    assert sorted(st['max']) == sorted('algo0_%d' % r for r in range(R))
    # without ini_pos_vel_att the first reference row is the initial state (the trajectory's own ini)
    fed2 = Sim([FS, 10.0, 0.0], str(tmp_path), ref_frame=0, imu=imu, algorithm=InsLoose(), seed=5, run_base=3)
    fed2.run(2)
    assert_close(fed2.get_data(['pos'])[0]['algo0_1'], b[1]['algo0_1'], 1e-9, 1e-4, 'ini from the reference rows')


@gpu
def test_reference_protocol_equals_run_batch(eng):
    """reset(); run(deepcopy([fs, gyro, accel, time, gps_time, gps])); get_results() per run, as
    InsAlgoMgr.run_algo drives a plugin: [pos, vel, att_euler, wb, ab], the rows of one run_batch."""
    from gnss_ins_sim_b200.ins_loose import InsLoose
    traj, imu, R = _traj(), _imu(), 3
    gyro, accel = eng.imu_noise(FS, R, eng.to_device(traj['ref_gyro']), eng.to_device(traj['ref_accel']),
                                imu.gyro_err, imu.accel_err, 8)
    gps = eng.gps_noise(R, eng.to_device(traj['ref_gps']), imu.gps_err, 0, 8).cpu().numpy()
    gyro, accel = gyro.cpu().numpy(), accel.cpu().numpy()
    batch = InsLoose(traj['ini'], imu=imu).run_batch(FS, gyro, accel, traj['time'], traj['gps_time'], gps)
    algo = InsLoose(traj['ini'], imu=imu)
    assert algo.output == ['pos', 'vel', 'att_euler', 'wb', 'ab']
    for r in range(R):
        algo.reset()
        algo.run(copy.deepcopy([FS, gyro[r], accel[r], traj['time'], traj['gps_time'], gps[r]]))
        out = algo.get_results()
        assert len(out) == 5
        for got, ref in zip(out, batch):
            assert got.shape == (traj['time'].size, 3) and np.array_equal(got, ref[r])


@gpu
def test_supplied_measurement_errors(eng):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.ins_loose import InsLoose
    from gnss_ins_sim_b200 import imu_model
    traj, imu = _traj(), _imu()
    n, m = traj['time'].size, traj['gps_time'].size
    algo = InsLoose(traj['ini'], imu=imu)
    g3, gps = np.zeros((2, n, 3)), np.tile(traj['ref_gps'], (2, 1, 1))
    with pytest.raises(ValueError, match=r'\[R, n, 3\]'):
        algo.run_batch(FS, g3, np.zeros((2, n - 1, 3)), traj['time'], traj['gps_time'], gps)
    with pytest.raises(ValueError, match=r'\[R, m, 6\]'):
        algo.run_batch(FS, g3, g3, traj['time'], traj['gps_time'], gps[:1])
    with pytest.raises(ValueError, match='gps_time needs one entry'):
        algo.run_batch(FS, g3, g3, traj['time'], traj['gps_time'][:-1], gps)
    with pytest.raises(ValueError, match='gps_visibility needs one entry'):
        algo.run_batch(FS, g3, g3, traj['time'], traj['gps_time'], gps, gps_visibility=np.ones(m + 1))
    bad = traj['gps_time'].copy()
    bad[5] = bad[4] + 0.001
    with pytest.raises(ValueError, match='land on IMU samples'):
        algo.run_batch(FS, g3, g3, traj['time'], bad, gps)
    with pytest.raises(ValueError, match='outside the IMU series'):
        algo.run_batch(FS, g3, g3, traj['time'], traj['gps_time'] + 20.0, gps)
    with pytest.raises(ValueError, match='needs ini_pos_vel_att'):
        InsLoose(imu=imu).run_batch(FS, g3, g3, traj['time'], traj['gps_time'], gps)
    other = imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True)
    with pytest.raises(ValueError, match="the Sim's imu"):
        Sim([FS, 10.0, 0.0], traj, ref_frame=0, imu=imu, algorithm=InsLoose(traj['ini'], imu=other)).run(2)
