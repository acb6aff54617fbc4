"""The loosely-coupled filter (K7) on vibrating sensors: random, sinusoidal and PSD vibration in its IMU
generator, through b2ins_ins_loose_ex_f64, engine.ins_loose and Sim(env=...).

The kernel is held to the spec (oracle/ekf_vib_np.py) on identical draws; without vibration the new entry
point is the old one; Sim hands env to every filter launch (experiment, history blocks, run blocks of the
PSD path); and at config-5 scale the InsLoose recipe for vibration keeps the filter consistent."""
import math
import os

import numpy as np
import pytest

from conftest import GOLDEN, load_golden, assert_close, wrap_pi
import ekf_vib_np

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
ENVS = {'random': ('[0.05 0.05 0.05]g-random', '[0.5 0.5 0.5]d-random'),
        'sinusoidal': ('[0.05 0.02 0.03]g-7.5Hz-sinusoidal', '[0.5 0.2 0.3]d-3Hz-sinusoidal'),
        'psd': (PSD, PSD * 1e-4),
        'random_acc_sinusoidal_gyro': ('[0.05 0.02 0.03]g-random', '[0.5 0.2 0.3]d-3Hz-sinusoidal')}


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _imu():
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True)


def _parse(kind):
    from gnss_ins_sim_b200.sim import parse_env
    acc, gyro = ENVS[kind]
    return parse_env(acc, FS), parse_env(gyro, FS)


def _turn_case():
    """The 90-degree-turn trajectory in ref_frame 0 with its 10 Hz GPS truth, all GPS samples visible."""
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    g = dict(load_golden('gps_90deg_rf0.npz'))
    g['gps_visibility'] = np.ones_like(g['gps_visibility'])
    nav = np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1)
    idx = np.rint(g['gps_time'] * 100.0).astype(np.int64)
    return t, g, nav, idx


def _launch(eng, t, g, nav, idx, imu, seed, runs, **kw):
    dev = [eng.to_device(a) for a in (t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'])]
    return eng.ins_loose(FS, runs, seed, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'], dev[0], dev[1],
                         dev[2], dev[3], torch.from_numpy(idx).cuda(),
                         eng.to_device(np.asarray(g['gps_visibility'], dtype=np.float64)), **kw)


def _vib_args(eng, kind, n, runs, seed, r0):
    """(device vib_accel, vib_gyro, spec vib_acc, vib_gyro): the parsed dicts, or for PSD the K5 series of
    exactly these runs, fed to both sides."""
    va, vg = _parse(kind)
    if kind != 'psd':
        return va, vg, va, vg
    (sa, na), (sg, ng) = (eng.psd_series(FS, n, runs, sensor, v, seed, run_offset=r0) for sensor, v in ((0, va), (1, vg)))
    return eng.vib_series(sa, na), eng.vib_series(sg, ng), sa.cpu().numpy(), sg.cpu().numpy()


@gpu
@pytest.mark.parametrize('kind', sorted(ENVS))
def test_kernel_equals_the_spec_with_vibration(eng, kind):
    """Same Philox draws (IMU noise and vibration, GPS noise, initial errors), 12 runs from run 5 (two 8-run
    CTAs): histories, bias estimates, end-point errors and the consistency record against the spec, with the
    tolerances of test_ekf.test_kernel_equals_the_spec."""
    t, g, nav, idx = _turn_case()
    imu = _imu()
    R, r0, seed = 12, 5, 2025
    n = t['ref_gyro'].shape[0]
    dva, dvg, sva, svg = _vib_args(eng, kind, n, R, seed, r0)
    o = ekf_vib_np.ins_loose(FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                             imu.gyro_err, imu.accel_err, imu.gps_err, seed, np.arange(r0, r0 + R), t['ini'],
                             vib_acc=sva, vib_gyro=svg, stats_start=100, want_hist=True)
    res = _launch(eng, t, g, nav, idx, imu, seed, R, run_offset=r0, stats_start=100, dump_runs=R, vel_rw=0.0,
                  vib_accel=dva, vib_gyro=dvg)
    quiet = _launch(eng, t, g, nav, idx, imu, seed, R, run_offset=r0, stats_start=100, vel_rw=0.0)
    assert np.abs(res.end_err.cpu().numpy() - quiet.end_err.cpu().numpy()).max() > 0.0
    att, pos, vel = res.att.cpu().numpy(), res.pos.cpu().numpy(), res.vel.cpu().numpy()
    assert np.abs(wrap_pi(att - o['att'])).max() < 1e-9
    assert_close(pos[:, :, :2], o['pos'][:, :, :2], 1e-9, 1e-4, 'lat/lon')
    assert_close(pos[:, :, 2], o['pos'][:, :, 2], 1e-9, 1e-2, 'alt')
    assert_close(vel, o['vel'], 1e-9, 1e-2, 'vel')
    assert_close(res.wb.cpu().numpy(), o['wb'], 1e-7, 1e-6, 'gyro bias estimate')
    assert_close(res.ab.cpu().numpy(), o['ab'], 1e-7, 1e-5, 'accel bias estimate')
    assert_close(res.end_err.cpu().numpy(), o['end_err'], 1e-7, 1e-6, 'end-point error')
    assert_close(res.end_bias.cpu().numpy(), o['end_bias'], 1e-7, 1e-6, 'end biases')
    con = res.consist.cpu().numpy()
    assert np.all(con[:, 18] == o['epochs'])
    assert_close(con[:, 0:3] / con[:, 18:19], o['nees'], 1e-6, 1e-3, 'NEES')
    assert np.abs(con[:, 3:18] / con[:, 18:19] - o['inside3']).max() < 1.5 / o['epochs']


@gpu
def test_no_vibration_entry_is_the_old_entry(eng, monkeypatch):
    """engine.ins_loose without vibration (b2ins_ins_loose_ex_f64 with VIB_NONE models), the new entry with
    NULL models and b2ins_ins_loose_f64 give the same bits."""
    t, g, nav, idx = _turn_case()
    imu = _imu()
    lib = eng._lib.load()

    class Entry(object):          # the library, with the ex entry replaced by `ex`
        def __init__(self, ex):
            self.b2ins_ins_loose_ex_f64 = ex

        def __getattr__(self, name):
            return getattr(lib, name)

    def outputs(ex=None):
        if ex is not None:
            monkeypatch.setattr(eng._lib, 'load', lambda: Entry(ex))
        r = _launch(eng, t, g, nav, idx, imu, 77, 13, run_offset=3, stats_start=100, dump_runs=5, dump_stride=3)
        monkeypatch.undo()
        return [x.cpu().numpy() for x in (r.end_err, r.end_bias, r.consist, r.att, r.pos, r.vel, r.wb, r.ab)]

    new = outputs()
    old = outputs(lambda cfg, vg, va, *rest: lib.b2ins_ins_loose_f64(cfg, *rest))
    null = outputs(lambda cfg, vg, va, *rest: lib.b2ins_ins_loose_ex_f64(cfg, None, None, *rest))
    for a, b, c in zip(new, old, null):
        assert np.array_equal(a, b) and np.array_equal(a, c)


@gpu
def test_argument_errors(eng):
    t, g, nav, idx = _turn_case()
    imu = _imu()
    bad = eng._lib.Vib()
    bad.type = 7
    with pytest.raises(ValueError, match='vib type 7'):
        _launch(eng, t, g, nav, idx, imu, 1, 4, vib_gyro=bad)
    no_series = eng._lib.Vib()
    no_series.type, no_series.series_len = eng._lib.VIB_SERIES, 16
    with pytest.raises(ValueError, match='VIB_SERIES needs series'):
        _launch(eng, t, g, nav, idx, imu, 1, 4, vib_accel=no_series)
    with pytest.raises(ValueError, match='VIB_SERIES needs series'):
        _launch(eng, t, g, nav, idx, imu, 1, 4, vib_accel={'type': 'psd'})


# ---- through Sim ----------------------------------------------------------------------------------------
def _sim(kind=None, **kw):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.ins_loose import InsLoose
    gm = load_golden('philox_90deg_mid_rf0.npz')
    gp = load_golden('gps_90deg_rf0.npz')
    traj = {k: gm[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro', 'ini')}
    traj.update(ref_gps=gp['ref_gps'], gps_time=gp['gps_time'], gps_visibility=np.ones_like(gp['gps_visibility']))
    env = None if kind is None else {'acc': ENVS[kind][0], 'gyro': ENVS[kind][1]}
    return Sim([FS, 10.0, 0.0], traj, ref_frame=0, imu=_imu(), env=env, algorithm=InsLoose(gm['ini']), seed=5,
               history_block=8, **kw)


def _results(sim):
    c = sim._mc[0]
    return c['end_err'], c['consist'], c['end_bias']


@gpu
@pytest.mark.parametrize('kind', ['random', 'sinusoidal', 'psd'])
def test_sim_env_reaches_the_filter(eng, kind):
    """env changes the filter's results, equals a direct engine.ins_loose call with the parsed model, and a
    history block of run r ends in the experiment launch's end state of r."""
    quiet, sim = _sim(), _sim(kind)
    quiet.run(20)
    sim.run(20)
    err, con, bias = _results(sim)
    assert not np.array_equal(err, _results(quiet)[0])
    d = sim._dev
    vg, va = sim._vib_pair(20, 0)            # (gyro, accel), as _ekf_launch takes them
    n = sim._traj['ref_gyro'].shape[0]
    start = int(round(min(30.0, 0.1 * n / FS) * FS))
    res = eng.ins_loose(FS, 20, 5, sim.imu.gyro_err, sim.imu.accel_err, sim.imu.gps_err, sim.algo[0].ini,
                        d['ref_gyro'], d['ref_accel'], d['ref_nav'], d['ref_gps'], d['gps_idx'], d['gps_vis'],
                        stats_start=start, vib_gyro=vg, vib_accel=va)
    if kind != 'psd':
        assert (va, vg) == _parse(kind)
    assert np.array_equal(res.end_err.cpu().numpy(), err) and np.array_equal(res.consist.cpu().numpy(), con)
    pos, vel, wb, ab = sim.get_data(['pos', 'vel', 'wb', 'ab'])
    for r in (0, 13, 19):          # history blocks [0, 8), [8, 16), [16, 20)
        k = 'algo0_%d' % r
        assert np.array_equal(wb[k][-1], bias[r, 0:3]) and np.array_equal(ab[k][-1], bias[r, 3:6])
        assert np.array_equal(pos[k][-1] - sim._traj['ref_pos'][-1], err[r, 3:6])
        assert np.array_equal(vel[k][-1] - sim._traj['ref_vel'][-1], err[r, 6:9])


@gpu
@pytest.mark.parametrize('kind', ['random', 'psd'])
def test_sim_run_base_split(eng, kind):
    """Runs 7..19 of one experiment are runs 0..12 of an experiment with run_base = 7."""
    whole, tail = _sim(kind), _sim(kind, run_base=7)
    whole.run(20)
    tail.run(13)
    for a, b in zip(_results(whole), _results(tail)):
        assert np.array_equal(a[7:], b)


@gpu
def test_sim_psd_run_blocks_equal_one_launch(eng, monkeypatch):
    one, blocks = _sim('psd'), _sim('psd')
    one.run(20)
    launches = []
    real = eng.ins_loose
    monkeypatch.setattr(eng, 'ins_loose', lambda *a, **k: launches.append((a[1], k['run_offset'])) or real(*a, **k))
    monkeypatch.setattr(blocks, '_allan_block', lambda *a: 6)
    blocks.run(20)
    assert launches == [(6, 0), (6, 6), (6, 12), (2, 18)]
    for a, b in zip(_results(one), _results(blocks)):
        assert np.array_equal(a, b)


@gpu
def test_config5_filter_with_vibration_at_scale(eng):
    """motion_def-ins.csv @100 Hz (n = 73 250), demo_ins_loose.py's IMU, 2048 runs, random vibration of 0.05 g
    and 0.5 deg/s: with the InsLoose recipe the NEES stays in test_config5_filter_is_consistent_at_scale's
    bands and >= 98.5 % of the errors inside 3 sigma; with the default model velocity and attitude are
    overconfident."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.ins_loose import InsLoose
    va, vg = _parse('random')
    dt = 1.0 / FS
    env = {'acc': ENVS['random'][0], 'gyro': ENVS['random'][1]}
    out = {}
    for label, algo in (('recipe', InsLoose(vel_model_std=math.sqrt(0.02 ** 2 + va['x'] ** 2 * dt),
                                            att_model_std=vg['x'] * math.sqrt(dt))),
                        ('default', InsLoose())):
        sim = Sim([FS, 10.0, 0.0], os.path.join(GOLDEN, 'motion_def-ins.csv'), ref_frame=0, imu=_imu(), env=env,
                  algorithm=algo, seed=5)
        sim.run(2048)
        c = sim.ekf_consistency()
        out[label] = (c['nees'].mean(0), c['inside3'].mean(0).min())
    print('config 5, random vibration, 2048 runs: NEES (pos, vel, att), min inside-3-sigma:', out)
    nees, inside = out['recipe']
    assert np.all(nees > 1.3) and np.all(nees < 3.8) and inside > 0.985, out
    nees, inside = out['default']
    assert nees[1] > 6.0 and nees[2] > 6.0, out
