"""The run-to-run turn-on bias in the loosely-coupled filter (K7) on the GPU: the RB forms of ekf_kernel through
b2ins_ins_loose_rx_f64 against the spec (oracle/ekf_rb_np.py), the forwarding of the older
entry points, the fed form's P0 (b2ins_ins_loose_fed_rx_f64), a saved experiment filtering back to itself, and
the filter's consistency at config-5 size with a turn-on bias that dominates the drift."""
import ctypes
import os

import numpy as np
import pytest

from conftest import GOLDEN, assert_close, wrap_pi
import ekf_proc_np
import ekf_rb_np
from test_ekf import DEMO_IMU, _turn_case

torch = pytest.importorskip('torch')
gpu = pytest.mark.gpu
FS = 100.0
R, R0, SEED = 12, 5, 2025
# gyro_b_std 100 deg/h and accel_b_std 0.02 m/s^2, well above the drift: the bias states have work to do
BIG = dict(DEMO_IMU, gyro_b_std=np.full(3, 100.0), accel_b_std=np.full(3, 0.02))


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _imu(acc=BIG):
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy=acc, axis=6, gps=True)


def _launch(eng, imu, t, g, nav, idx, runs=R, run_offset=R0, **kw):
    dev = [eng.to_device(a) for a in (t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'])]
    return eng.ins_loose(FS, runs, SEED, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'], *dev,
                         torch.from_numpy(idx).cuda(), eng.to_device(np.asarray(g['gps_visibility'], dtype=np.float64)),
                         run_offset=run_offset, vel_rw=kw.pop('vel_rw', 0.0), **kw)


def _check(res, o, what):
    """test_ekf.py::test_kernel_equals_the_spec's tolerances on histories (NaN where the spec has NaN), bias
    estimates, end_err, end_bias, end_bias_err and the consistency record."""
    att, pos, vel = res.att.cpu().numpy(), res.pos.cpu().numpy(), res.vel.cpu().numpy()
    for k, got in (('att', att), ('pos', pos), ('vel', vel)):
        assert np.array_equal(np.isnan(got), np.isnan(o[k])), what + ' NaN rows of ' + k
    ok, oka = ~np.isnan(o['pos'][:, :, 0]), ~np.isnan(o['att'][:, :, 0])
    assert np.abs(wrap_pi(att[oka] - o['att'][oka])).max() < 1e-9, what
    assert_close(pos[ok][:, :2], o['pos'][ok][:, :2], 1e-9, 1e-4, what + ' lat/lon')
    assert_close(pos[ok][:, 2], o['pos'][ok][:, 2], 1e-9, 1e-2, what + ' alt')
    assert_close(vel[ok], o['vel'][ok], 1e-9, 1e-2, what + ' vel')
    assert_close(res.wb.cpu().numpy(), o['wb'], 1e-7, 1e-6, what + ' gyro bias estimate')
    assert_close(res.ab.cpu().numpy(), o['ab'], 1e-7, 1e-5, what + ' accel bias estimate')
    assert_close(res.end_err.cpu().numpy(), o['end_err'], 1e-7, 1e-6, what + ' end-point error')
    assert_close(res.end_bias.cpu().numpy(), o['end_bias'], 1e-7, 1e-6, what + ' end biases')
    assert_close(res.end_bias_err.cpu().numpy(), o['end_bias_err'], 1e-7, 1e-6, what + ' end bias errors')
    con = res.consist.cpu().numpy()
    assert np.all(con[:, 18] == o['epochs']), what
    assert_close(con[:, 0:3] / con[:, 18:19], o['nees'], 1e-6, 1e-3, what + ' NEES')
    assert np.abs(con[:, 3:18] / con[:, 18:19] - o['inside3']).max() < 1.5 / o['epochs'], what


@gpu
@pytest.mark.parametrize('form', ['plain', 'random_vib', 'proc_ned', 'align_gps'])
def test_kernel_equals_the_spec(eng, form):
    """The RB forms against the spec on identical draws (IMU, GPS, initial state and turn-on bias), 12 runs from
    run 5 on the 90-degree turn."""
    from gnss_ins_sim_b200.sim import parse_env
    t, g, nav, idx = _turn_case()
    imu = _imu()
    args = (FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'], imu.gyro_err,
            imu.accel_err, imu.gps_err, SEED, np.arange(R0, R0 + R))
    kw = {}
    if form == 'random_vib':
        va, vg = parse_env('[0.05 0.05 0.05]g-random', FS), parse_env('[0.5 0.5 0.5]d-random', FS)
        o = ekf_rb_np.ins_loose(*args, t['ini'], vib_acc=va, vib_gyro=vg, stats_start=100, want_hist=True)
        kw = dict(vib_accel=va, vib_gyro=vg)
    elif form == 'align_gps':
        o = ekf_rb_np.ins_loose_aligned(*args, 'gps', stats_start=100, want_hist=True, ini_att_std=(0.02, 0.005, 0.15))
        kw = dict(align=('gps', 0.15 ** 2), ini_att_std=(0.02, 0.005, 0.15))
    else:
        o = ekf_rb_np.ins_loose(*args, t['ini'], stats_start=100, want_hist=True)
        if form == 'proc_ned':
            kw = dict(proc_start=333, proc_pos_frame=1)
    res = _launch(eng, imu, t, g, nav, idx, stats_start=100, dump_runs=R, bias_err=True, **kw)
    _check(res, o, form)
    if form == 'proc_ned':
        ref = ekf_proc_np.process_stats(o['att'], o['pos'], o['vel'], nav, 333, 'ned')
        ps = res.proc_stats.cpu().numpy()
        assert np.abs(ps[:, :, 0:3] - ref[:, :, 0:3]).max() < 1e-9
        assert np.abs(ps[:, :, 3:6] - ref[:, :, 3:6]).max() < 1e-4
        assert np.abs(ps[:, :, 6:9] - ref[:, :, 6:9]).max() < 1e-7
    # the runs' biases are the run-error table's (Sim.imu_run_errors draws them through the same device function)
    tab = eng.imu_run_errors(R, imu.gyro_err, imu.accel_err, SEED, run_offset=R0).cpu().numpy()
    assert_close(tab[:, 1, :, 3], ekf_rb_np.turn_on_bias(imu.gyro_err, 1, SEED, np.arange(R0, R0 + R)) -
                 imu.gyro_err['b'], 1e-13, 0.0, form + ' gyro b_run')


def _outputs(res):
    return {k: getattr(res, k).cpu().numpy() for k in ('end_err', 'end_bias', 'consist', 'att', 'pos', 'vel', 'wb', 'ab')}


@gpu
def test_forwarding_is_bit_for_bit(eng):
    """b2ins_ins_loose_f64 (which forwards to _rx with nulls) and engine.ins_loose (_rx with null run errors) give
    the same bits; the RB form with zero sigmas gives the plain form's outputs bit for bit, plus end_bias_err."""
    from gnss_ins_sim_b200 import _lib
    t, g, nav, idx = _turn_case()
    imu = _imu(DEMO_IMU)
    plain = _launch(eng, imu, t, g, nav, idx, stats_start=100, dump_runs=R)
    assert plain.end_bias_err is None
    dev = [eng.to_device(a) for a in (t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'])]
    d_idx, d_vis = torch.from_numpy(idx).cuda(), eng.to_device(np.asarray(g['gps_visibility'], dtype=np.float64))
    n = t['ref_gyro'].shape[0]
    cfg = eng._ekf_config(FS, n, R, g['ref_gps'].shape[0], SEED, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'],
                          R0, (0.02, 0.005, 0.005), True, 100, R, 1, 0.0, 0.0)
    old = {'end_err': torch.empty(R, 9, dtype=torch.float64, device='cuda'),
           'end_bias': torch.empty(R, 6, dtype=torch.float64, device='cuda'),
           'consist': torch.empty(R, 19, dtype=torch.float64, device='cuda')}
    old.update({k: torch.empty(R, n, 3, dtype=torch.float64, device='cuda') for k in ('att', 'pos', 'vel', 'wb', 'ab')})
    p = lambda a: ctypes.c_void_p(a.data_ptr())      # noqa: E731
    _lib.check(_lib.load().b2ins_ins_loose_f64(
        ctypes.byref(cfg), *[p(a) for a in dev], p(d_idx), p(d_vis),
        *[p(old[k]) for k in ('end_err', 'end_bias', 'consist', 'att', 'pos', 'vel', 'wb', 'ab')],
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    got = _outputs(plain)
    for k, v in old.items():
        assert np.array_equal(v.cpu().numpy(), got[k], equal_nan=True), k
    rb = _launch(eng, imu, t, g, nav, idx, stats_start=100, dump_runs=R, bias_err=True)
    for k, v in _outputs(rb).items():
        assert np.array_equal(v, got[k], equal_nan=True), k
    o = ekf_rb_np.ins_loose(FS, t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'], idx, g['gps_visibility'],
                         imu.gyro_err, imu.accel_err, imu.gps_err, SEED, np.arange(R0, R0 + R), t['ini'],
                         stats_start=100)
    assert_close(rb.end_bias_err.cpu().numpy(), o['end_bias_err'], 1e-7, 1e-6, 'end bias errors, zero sigma')


@gpu
def test_fed_rx_reproduces_the_generated_rb_run(eng):
    """K1-rx's and K6's measurements of the same runs, with the same initial draw, through the fed form whose P0
    knows b_std, filter to the generated RB experiment at test_gpu_ekf_fed.py's tolerances: K7 drew the biases
    K1 draws, which are Sim.imu_run_errors()'s."""
    from test_gpu_ekf_fed import _close, _host
    t, g, nav, idx = _turn_case()
    imu = _imu()
    runs, r0, seed = 21, 7, 4711
    vis = np.ones(idx.size)
    vis[30:40] = 0.0
    ref = [eng.to_device(a) for a in (t['ref_gyro'], t['ref_accel'], nav, g['ref_gps'])]
    d_idx, d_vis = torch.from_numpy(idx).cuda(), eng.to_device(vis)
    gen = eng.ins_loose(FS, runs, seed, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'], *ref, d_idx, d_vis,
                        run_offset=r0, dump_runs=runs, bias_err=True)
    gyro, accel = eng.imu_noise(FS, runs, ref[0], ref[1], imu.gyro_err, imu.accel_err, seed, run_offset=r0)
    gps = eng.gps_noise(runs, ref[3], imu.gps_err, 0, seed, run_offset=r0)
    fed = eng.ins_loose_fed(FS, gyro, accel, gps, d_idx, d_vis, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'],
                            seed=seed, ini_draw=True, run_offset=r0, ref_nav=ref[2], dump_runs=runs)
    print('largest |fed - generated| with a turn-on bias:', _close(_host(fed), _host(gen), 'fed vs generated'))
    # without b_std in the fed model's P0 the same data filter differently
    bare = eng.ins_loose_fed(FS, gyro, accel, gps, d_idx, d_vis, *[{k: v for k, v in e.items() if k != 'b_std'}
                                                                      for e in (imu.gyro_err, imu.accel_err)],
                             imu.gps_err, t['ini'], seed=seed, ini_draw=True, run_offset=r0, ref_nav=ref[2])
    assert np.abs(bare.end_bias.cpu().numpy() - gen.end_bias.cpu().numpy()).max() > 1e-6


@gpu
def test_saved_rb_experiment_filters_back_to_itself(eng, tmp_path):
    """A generated experiment with a turn-on bias written with save_data and read back as a logged-data directory,
    with the same seed and run_base: the same histories and end-point errors (the fed filter's P0 takes b_std)."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.ins_loose import InsLoose
    from test_gpu_ekf_fed import _close, _traj
    traj, imu, runs = _traj(), _imu(), 11
    gen = Sim([FS, 10.0, 0.0], traj, ref_frame=0, imu=imu, algorithm=InsLoose(traj['ini'], imu=imu), seed=5,
              run_base=3)
    gen.run(runs)
    c = gen.ekf_consistency()
    assert c['bias_err'].shape == (runs, 6) and np.all(np.isfinite(c['bias_err']))
    gen.save_data(str(tmp_path), names=['time', 'gyro', 'accel', 'gps', 'gps_time', 'gps_visibility', 'ref_pos',
                                        'ref_vel', 'ref_att_euler'])
    fed = Sim([FS, 10.0, 0.0], str(tmp_path), ref_frame=0, algorithm=InsLoose(traj['ini'], imu=imu), seed=5,
              run_base=3)
    fed.run(runs)
    names = ['att_euler', 'pos', 'vel', 'wb', 'ab']
    a, b = gen.get_data(names), fed.get_data(names)
    for r in range(runs):
        key = 'algo0_%d' % r
        _close({k: b[i][key] for i, k in enumerate(('att', 'pos', 'vel', 'wb', 'ab'))},
               {k: a[i][key] for i, k in enumerate(('att', 'pos', 'vel', 'wb', 'ab'))}, key)
    assert_close(fed.end_point_errors(), gen.end_point_errors(), 1e-7, 1e-6, 'end-point errors')
    assert_close(fed._mc[0]['end_bias'], gen._mc[0]['end_bias'], 1e-7, 1e-6, 'end biases')
    # the biases the experiment drew are Sim.imu_run_errors()'s: the estimates end near them
    b_run = gen.imu_run_errors()
    truth_minus_drift = c['end_bias'] - c['bias_err']
    drift = truth_minus_drift - np.concatenate([b_run['gyro'][:, :, 3], b_run['accel'][:, :, 3]], axis=1)
    assert np.abs(drift[:, 3:]).max() < 10 * 8.02e-5        # accel: what is left is the Gauss-Markov drift


@gpu
def test_config5_filter_with_a_turn_on_bias_at_scale(eng):
    """motion_def-ins.csv @100 Hz (n = 73 250), demo_ins_loose.py's IMU plus gyro_b_std 10 deg/h and accel_b_std
    5e-4 m/s^2 (the drift: 3.5 deg/h and <= 8e-5 m/s^2), 2048 runs through Sim.

    What holds at this length: the position and velocity blocks keep test_ekf.py's
    test_config5_filter_is_consistent_at_scale bounds (NEES 2.96 and 1.74, >= 99.3 % inside 3 sigma, on an H100),
    and no axis ends with a bias error wider than its prior spread, sqrt(b_std^2 + drift^2), beyond sampling.
    What does not: the filter's bias model is first-order Gauss-Markov (tau 100 s gyro, 200 s accel), so over
    732 s it lets the constant turn-on bias decay out of the bias states.  Measured: attitude NEES 6.0, bias
    states inside 3 sigma in 79-88 % (gyro) and 50-58 % (accel) of epochs, and bias_err std / b_std of
    0.55 / 0.54 / 0.86 (gyro) and 1.00 / 1.00 / 0.96 (accel).  Those figures are printed, not asserted:
    DESIGN.md section 10 keeps a constant-bias model for long runs open."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.ins_loose import InsLoose
    imu = _imu(dict(DEMO_IMU, gyro_b_std=np.full(3, 10.0), accel_b_std=np.full(3, 5e-4)))
    sim = Sim([100.0, 10.0, 0.0], os.path.join(GOLDEN, 'motion_def-ins.csv'), ref_frame=0, imu=imu,
              algorithm=InsLoose(), seed=5)
    sim.run(2048)
    c = sim.ekf_consistency()
    nees = c['nees'].mean(0)
    inside = c['inside3'].mean(0)
    sig = np.concatenate([imu.gyro_err['b_std'], imu.accel_err['b_std']])
    drift = np.concatenate([imu.gyro_err['b_drift'], imu.accel_err['b_drift']])
    spread = c['bias_err'].std(0) / sig
    print('mean NEES', nees, 'inside 3 sigma', inside, 'bias_err std / b_std (gyro xyz, accel xyz)', spread)
    assert c['bias_err'].shape == (2048, 6) and np.all(np.isfinite(c['bias_err']))
    assert np.all(nees[0:2] > 1.3) and np.all(nees[0:2] < 3.8), nees
    assert inside[0:6].min() > 0.985, inside
    assert np.all(c['bias_err'].std(0) < 1.1 * np.sqrt(sig ** 2 + drift ** 2)), spread
