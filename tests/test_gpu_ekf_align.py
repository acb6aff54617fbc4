"""The self-initialising loosely-coupled filter on the GPU: b2ins_ins_loose_align_f64 and _fed_align_f64 through
engine.ins_loose / ins_loose_fed and InsLoose(align_yaw=...).

The generated aligned kernel is held to the spec (oracle/ekf_align_np.py) on identical draws, with the tolerances of
test_gpu_ekf_vib.py / test_gpu_ekf_proc.py; the fed form on the same measurements equals the generated form; align
off through the new entry point is the existing entry point bit for bit."""
import ctypes

import numpy as np
import pytest

from conftest import load_golden, assert_close, wrap_pi
import ekf_align_np
import ekf_proc_np

torch = pytest.importorskip('torch')
gpu = pytest.mark.gpu
FS = 100.0
DEMO_IMU = {'gyro_b': np.zeros(3), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
            'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
            'accel_b': np.zeros(3), 'accel_vrw': np.array([0.03119, 0.03009, 0.04779]),
            'accel_b_stability': np.array([4.29e-5, 5.72e-5, 8.02e-5]),
            'accel_b_corr': np.array([200.0, 200.0, 200.0])}       # demo_ins_loose.py:28-37
R, R0, SEED = 12, 5, 2025


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _imu():
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True)


def _turn(first_visible=1.0):
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    g = dict(load_golden('gps_90deg_rf0.npz'))
    g['gps_visibility'] = (g['gps_time'] >= first_visible).astype(np.float64)
    nav = np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1)
    return t, g, nav, np.rint(g['gps_time'] * FS).astype(np.int64)


def _launch(eng, t, g, nav, idx, imu, **kw):
    dev = [eng.to_device(a) for a in (t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'])]
    return eng.ins_loose(FS, R, SEED, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'], dev[0], dev[1], dev[2],
                         dev[3], torch.from_numpy(idx).cuda(), eng.to_device(g['gps_visibility']), run_offset=R0,
                         vel_rw=0.0, **kw)


def _check_hist(res, o):
    att, pos, vel = (getattr(res, k).cpu().numpy() for k in ('att', 'pos', 'vel'))
    for a, b in ((att, o['att']), (pos, o['pos']), (vel, o['vel'])):
        assert np.array_equal(np.isnan(a), np.isnan(b))
    ok = ~np.isnan(o['pos'][:, :, 0])
    oka = ~np.isnan(o['att'][:, :, 0])
    assert np.abs(wrap_pi(att[oka] - o['att'][oka])).max() < 1e-9
    assert_close(pos[ok][:, :2], o['pos'][ok][:, :2], 1e-9, 1e-4, 'lat/lon')
    assert_close(pos[ok][:, 2], o['pos'][ok][:, 2], 1e-9, 1e-2, 'alt')
    assert_close(vel[ok], o['vel'][ok], 1e-9, 1e-2, 'vel')
    assert_close(res.wb.cpu().numpy(), o['wb'], 1e-7, 1e-6, 'gyro bias estimate')
    assert_close(res.ab.cpu().numpy(), o['ab'], 1e-7, 1e-5, 'accel bias estimate')


@gpu
@pytest.mark.parametrize('yaw', [-0.7, 'gps'])
@pytest.mark.parametrize('vib', [None, 'random'])
@pytest.mark.parametrize('first_visible', [0.0, 1.0])
def test_kernel_equals_the_spec(eng, yaw, vib, first_visible):
    """Histories (NaN mask identical), bias estimates, end-point errors and the consistency record of 12 runs from
    run 5 against the spec on identical draws; the fix row at sample 0 (start at sample 9) or after the invisible
    first second."""
    from gnss_ins_sim_b200.sim import parse_env
    t, g, nav, idx = _turn(first_visible)
    imu = _imu()
    va = vg = None
    if vib:
        va, vg = parse_env('[0.05 0.05 0.05]g-random', FS), parse_env('[0.5 0.5 0.5]d-random', FS)
    o = ekf_align_np.ins_loose_gen(FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                                   imu.gyro_err, imu.accel_err, imu.gps_err, SEED, np.arange(R0, R0 + R), yaw,
                                   vib_acc=va, vib_gyro=vg, stats_start=100, want_hist=True,
                                   ini_att_std=(0.02, 0.005, 0.15))
    res = _launch(eng, t, g, nav, idx, imu, stats_start=100, dump_runs=R, vib_accel=va, vib_gyro=vg,
                  align=(yaw, 0.15 ** 2))
    assert res.start == o['start']
    _check_hist(res, o)
    assert_close(res.end_err.cpu().numpy(), o['end_err'], 1e-7, 1e-6, 'end-point error')
    assert_close(res.end_bias.cpu().numpy(), o['end_bias'], 1e-7, 1e-6, 'end biases')
    con = res.consist.cpu().numpy()
    assert np.all(con[:, 18] == o['epochs'])
    assert_close(con[:, 0:3] / con[:, 18:19], o['nees'], 1e-6, 1e-3, 'NEES')
    assert np.abs(con[:, 3:18] / con[:, 18:19] - o['inside3']).max() < 1.5 / o['epochs']


@gpu
@pytest.mark.parametrize('frame', [0, 1, 2])
@pytest.mark.parametrize('start', [0, 500])
def test_proc_statistics_start_at_the_fix(eng, frame, start):
    """PROC statistics of the aligned kernel against the spec's histories from max(start, fix sample)."""
    t, g, nav, idx = _turn(1.0)
    imu = _imu()
    o = ekf_align_np.ins_loose_gen(FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                                   imu.gyro_err, imu.accel_err, imu.gps_err, SEED, np.arange(R0, R0 + R), 'gps',
                                   want_hist=True)
    res = _launch(eng, t, g, nav, idx, imu, align=('gps', 0.0), proc_start=start, proc_pos_frame=frame)
    ref = ekf_proc_np.process_stats(o['att'], o['pos'], o['vel'], nav, max(start, o['start']),
                                    ekf_proc_np.FRAMES[frame])
    ps = res.proc_stats.cpu().numpy()
    assert np.all(np.isfinite(ps))
    assert np.abs(ps[:, :, 0:3] - ref[:, :, 0:3]).max() < 1e-9
    assert np.abs(ps[:, :, 3:6] - ref[:, :, 3:6]).max() < (1e-10 if frame == 0 else 1e-4)
    assert np.abs(ps[:, :, 6:9] - ref[:, :, 6:9]).max() < 1e-7


@gpu
@pytest.mark.parametrize('yaw', [-0.7, 'gps'])
def test_fed_aligned_equals_generated_aligned(eng, yaw):
    """The generated experiment's own measurements (the spec's, identical draws) through the fed aligned kernel:
    the generated aligned kernel's histories and end-point errors."""
    t, g, nav, idx = _turn(1.0)
    imu = _imu()
    o = ekf_align_np.ins_loose_gen(FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                                   imu.gyro_err, imu.accel_err, imu.gps_err, SEED, np.arange(R0, R0 + R), yaw,
                                   want_imu=True)
    gen = _launch(eng, t, g, nav, idx, imu, dump_runs=R, align=(yaw, 0.15 ** 2))
    fed = eng.ins_loose_fed(FS, eng.to_device(o['gyro']), eng.to_device(o['accel']), eng.to_device(o['gps']),
                            torch.from_numpy(idx).cuda(), eng.to_device(g['gps_visibility']), imu.gyro_err,
                            imu.accel_err, imu.gps_err, None, ref_nav=eng.to_device(nav), dump_runs=R, vel_rw=0.0,
                            align=(yaw, 0.15 ** 2))
    assert fed.start == gen.start
    for k in ('att', 'pos', 'vel'):
        a, b = getattr(fed, k).cpu().numpy(), getattr(gen, k).cpu().numpy()
        assert np.array_equal(np.isnan(a), np.isnan(b))
        d = np.nan_to_num(a - b)
        assert np.abs(wrap_pi(d) if k == 'att' else d).max() < (1e-9 if k == 'pos' else 1e-7), k
    assert np.abs(fed.end_err.cpu().numpy() - gen.end_err.cpu().numpy()).max() < 1e-7


@gpu
def test_align_off_is_the_existing_entry_point(eng):
    """b2ins_ins_loose_align_f64 with B2INS_ALIGN_OFF gives the bits of b2ins_ins_loose_ex_f64."""
    from gnss_ins_sim_b200 import _lib
    t, g, nav, idx = _turn(1.0)
    imu = _imu()
    old = _launch(eng, t, g, nav, idx, imu, dump_runs=R, stats_start=100)
    new = _launch(eng, t, g, nav, idx, imu, dump_runs=R, stats_start=100)
    for k in ('end_err', 'end_bias', 'consist', 'att', 'pos', 'vel', 'wb', 'ab'):
        getattr(new, k).zero_()
    n, m = t['ref_gyro'].shape[0], g['ref_gps'].shape[0]
    cfg = eng._ekf_config(FS, n, R, m, SEED, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'], R0,
                          (0.02, 0.005, 0.005), True, 100, R, 1, 0.0, 0.0)
    dev = [eng.to_device(a) for a in (t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'])]
    gi, gv = torch.from_numpy(idx).cuda(), eng.to_device(g['gps_visibility'])
    off = _lib.EkfAlign()
    p = eng._ptr
    _lib.check(_lib.load().b2ins_ins_loose_align_f64(
        ctypes.byref(cfg), ctypes.byref(off), None, None, -1, 0, p(dev[0]), p(dev[1]), p(dev[2]), p(dev[3]),
        ctypes.c_void_p(gi.data_ptr()), p(gv), p(new.end_err), p(new.end_bias), p(new.consist), None, p(new.att),
        p(new.pos), p(new.vel), p(new.wb), p(new.ab), eng._stream()))
    torch.cuda.synchronize()
    for k in ('end_err', 'end_bias', 'consist', 'att', 'pos', 'vel', 'wb', 'ab'):
        assert torch.equal(getattr(old, k), getattr(new, k)), k


@gpu
def test_insloose_run_and_run_batch_without_ini(eng):
    """InsLoose(imu=..., align_yaw='gps') filters supplied measurements with no initial state: run_batch equals
    the spec's fed form, run() its first run."""
    from gnss_ins_sim_b200.ins_loose import InsLoose
    t, g, nav, idx = _turn(1.0)
    imu = _imu()
    o = ekf_align_np.ins_loose_gen(FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                                   imu.gyro_err, imu.accel_err, imu.gps_err, SEED, np.arange(4), 'gps',
                                   want_imu=True, want_hist=True, vel_rw=0.02)
    time = np.arange(t['ref_gyro'].shape[0]) / FS
    algo = InsLoose(imu=imu, align_yaw='gps')
    pos, vel, att, wb, ab = algo.run_batch(FS, o['gyro'], o['accel'], time, g['gps_time'], o['gps'],
                                           gps_visibility=g['gps_visibility'])
    assert np.array_equal(np.isnan(pos), np.isnan(o['pos']))
    ok = ~np.isnan(o['pos'])
    assert np.abs(pos[ok] - o['pos'][ok]).max() < 1e-4
    algo.run([FS, o['gyro'][0], o['accel'][0], time, g['gps_time'][10:], o['gps'][0, 10:]])
    out = algo.get_results()
    assert out[0].shape == (time.size, 3) and np.isfinite(out[0][-1]).all()
    with pytest.raises(ValueError):
        InsLoose(imu=imu, align_yaw='gps').run_batch(FS, o['gyro'], o['accel'], time, g['gps_time'], o['gps'],
                                                     gps_visibility=np.zeros(len(g['gps_time'])))


# ---- through Sim ------------------------------------------------------------------------------------------------
def _sim_traj():
    """The 90-degree turn of test_gpu_ekf_fed.py's Sim tests: every GPS row visible but rows 40..51."""
    gm = load_golden('philox_90deg_mid_rf0.npz')
    gp = load_golden('gps_90deg_rf0.npz')
    traj = {k: gm[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro', 'ini')}
    traj.update(ref_gps=gp['ref_gps'], gps_time=gp['gps_time'], gps_visibility=np.ones_like(gp['gps_visibility']))
    traj['gps_visibility'][40:52] = 0.0
    return traj


def _hist_close(a, b, what):
    """Histories read back from text files: the same NaN rows, values within test_gpu_ekf_fed.py's bounds."""
    assert np.array_equal(np.isnan(a), np.isnan(b)), what
    ok = ~np.isnan(b)
    d = np.abs(a[ok] - b[ok])
    return float(d.max()) if d.size else 0.0


@gpu
def test_saved_aligned_experiment_filters_back_without_reference_files(eng, tmp_path):
    """A generated aligned experiment written with save_data, its ref_* files left out, filters back through
    Sim(<dir>) to the generated histories; with the reference files its process statistics start at the fix
    sample (finite), as the generated experiment's do.  The trajectory's initial state is not used."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.ins_loose import InsLoose
    traj, imu, Rn = _sim_traj(), _imu(), 6
    gen = Sim([FS, 10.0, 0.0], traj, ref_frame=0, imu=imu, algorithm=InsLoose(imu=imu, align_yaw='gps'), seed=5,
              run_base=3)
    gen.run(Rn)
    names = ['att_euler', 'pos', 'vel', 'wb', 'ab']
    a = gen.get_data(names)
    assert np.isnan(a[1]['algo0_0'][0]).all() and np.isfinite(a[1]['algo0_0'][-1]).all()
    ps_gen = gen.get_error_stats('pos', 0.0, extra_opt='ned')
    assert all(np.isfinite(v).all() for v in ps_gen['std'].values())
    gen.save_data(str(tmp_path), names=['time', 'gyro', 'accel', 'gps', 'gps_time', 'gps_visibility'])
    assert not list(tmp_path.glob('ref_*'))
    fed = Sim([FS, 10.0, 0.0], str(tmp_path), ref_frame=0, imu=imu, algorithm=InsLoose(align_yaw='gps'), seed=5)
    fed.run(Rn)
    b = fed.get_data(names)
    assert fed.end_point_errors() is None
    for r in range(Rn):
        key = 'algo0_%d' % r
        assert _hist_close(b[0][key], a[0][key], 'att') < 1e-6
        assert _hist_close(b[1][key][:, :2], a[1][key][:, :2], 'lat/lon') < 1e-9
        assert _hist_close(b[1][key][:, 2], a[1][key][:, 2], 'alt') < 1e-3
        assert _hist_close(b[2][key], a[2][key], 'vel') < 1e-4
        for i in (3, 4):
            assert _hist_close(b[i][key], a[i][key], names[i]) < 1e-6
    assert_close(fed._mc[0]['end_bias'], gen._mc[0]['end_bias'], 1e-6, 1e-6, 'end biases')
    # with the reference files the host statistics of the logged path start at the fix sample too
    gen.save_data(str(tmp_path), names=['ref_pos', 'ref_vel', 'ref_att_euler'])
    ref = Sim([FS, 10.0, 0.0], str(tmp_path), ref_frame=0, imu=imu, algorithm=InsLoose(align_yaw='gps'), seed=5)
    ref.run(Rn)
    assert ref._mc[0]['start'] == 9             # GPS row 0 is visible: the fix is at sample 9, rows 0..8 are NaN
    ps = ref.get_error_stats('pos', 0.0, extra_opt='ned')
    for k in ('max', 'avg', 'std'):
        for key, v in ps[k].items():
            assert np.isfinite(v).all(), (k, key)
            assert_close(v, ps_gen[k][key], 1e-3, 1.0, 'pos %s %s' % (k, key))     # metres: text-file ulps
    assert np.isfinite(ref.end_point_errors()).all()


@gpu
def test_aligned_filter_is_consistent_at_scale(eng):
    """motion_def-ins.csv @100 Hz (n = 73 250), demo_ins_loose.py's IMU, 2048 runs aligned from rest with a given
    heading 0.1 rad (the truth is 0) and ini_att_std[2] = 0.15: over the GPS epochs from 300 s (after the first
    acceleration) the NEES and the inside-3-sigma fractions meet test_ekf.py's bounds for the truth-initialised
    filter (NEES 1.3 .. 3.8 per block, >= 98.5 % inside 3 sigma), and stay near the truth-initialised filter's
    own figures on the same runs."""
    import os
    from conftest import GOLDEN
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.ins_loose import InsLoose
    imu = _imu()
    out = {}
    for kind, algo in (('truth', InsLoose(ini_att_std=(0.02, 0.005, 0.15))),
                       ('aligned', InsLoose(ini_att_std=(0.02, 0.005, 0.15), align_yaw=0.1))):
        sim = Sim([100.0, 10.0, 0.0], os.path.join(GOLDEN, 'motion_def-ins.csv'), ref_frame=0, imu=imu,
                  algorithm=algo, seed=5)
        sim.run(8)
        res = sim._ekf_launch(algo, 0, 2048, stats_start=30000)
        c = res.consist.cpu().numpy()
        out[kind] = (c[:, 0:3].sum(0) / c[:, 18].sum(), (c[:, 3:18] / c[:, 18:19]).mean(0),
                     res.end_err.cpu().numpy())
    print('NEES (pos, vel, att) truth %s aligned %s; min inside-3-sigma truth %.4f aligned %.4f'
          % (out['truth'][0], out['aligned'][0], out['truth'][1].min(), out['aligned'][1].min()))
    nees, inside, end = out['aligned']
    assert np.all(nees > 1.3) and np.all(nees < 3.8), nees
    assert inside.min() > 0.985, inside
    assert np.all(np.abs(nees - out['truth'][0]) < 0.5), (nees, out['truth'][0])
    assert np.all(np.isfinite(end))
    assert np.abs(wrap_pi(end[:, 0])).max() < 0.05           # the heading has converged from its 0.1 rad error
