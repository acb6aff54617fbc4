"""Allan noise identification (K13, engine.allan_fit) on the GPU: against the NumPy oracle (oracle/allan_fit_np.py)
on K4, K4o and fused K1+K4 curves in every addressing, model curves of all 31 supports and the edge rules; the
same bits whatever the batch and position; the laws of white noise, a rate random walk, a rate ramp and
quantisation through Sim and logged directories, held to the oracle's envelopes; Sim's fused, materialised and
vibration paths against engine.allan_fit, and save_data."""
import os

import numpy as np
import pytest

import allan_fit_np as af
import oracle_np

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

FS, N = 100.0, 360000


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _coef(out):
    """The coefficients C_-2 .. C_2 behind six outputs."""
    q, nn, b, k, r = out[:5]
    return np.array([3.0 * q * q, nn * nn, (b / af.B_SCALE) ** 2, k * k / 3.0, r * r / 2.0])


def _clear(info):
    """The oracle's choice is away from ties: every other feasible support is worse by > 1e-9 of sum w, or ties it
    (within 1e-15 of sum w: a superset of an exact fit)."""
    d = np.array([o - info['objective'] for m, o in info['objectives'].items() if m != info['mask']])
    return np.all((d > 1e-9 * info['W']) | (np.abs(d) < 1e-15 * info['W']))


def _check(got, var, n, fs, what, need_clear=True):
    """got [S, 6] (device outputs) against the oracle on var [S, ntau]: the same support, the fitted model to 1e-10
    relative per bin, the coefficients to 1e-9 relative and B_min to 1e-12.  need_clear: the fixture is away from
    support ties (_clear) for every series, so that the support is decided."""
    for s, v in enumerate(var):
        o, info = af.fit(v, n, fs, detail=True)
        if np.isnan(o).all():
            assert np.isnan(got[s]).all(), (what, s)
            continue
        if need_clear:
            assert _clear(info), (what, s, info['mask'])
        assert abs(got[s][5] - o[5]) <= 1e-12 * o[5], (what, s)
        C, Cg = info['C'], _coef(got[s])
        assert np.array_equal(C > 0.0, Cg > 0.0), (what, s, C, Cg)
        assert np.all(np.abs(Cg - C) <= 1e-9 * C), (what, s, np.abs(Cg - C) / np.where(C > 0, C, 1.0))
        mo, mg = af.model_curve(C, n, fs), af.model_curve(Cg, n, fs)
        assert np.all(np.abs(mg - mo) <= 1e-10 * mo), (what, s)


def _fit(eng, n, var, **kw):
    out = eng.allan_fit(FS, n, var, **kw)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _series(seed, S, n):
    rng = np.random.default_rng(seed)
    x = 1e-3 * np.sqrt(FS) * rng.standard_normal((S, n))
    x += np.cumsum(rng.uniform(1e-5, 1e-4, (S, 1)) / np.sqrt(FS) * rng.standard_normal((S, n)), axis=1)
    x += rng.uniform(0.0, 2e-6, (S, 1)) * np.arange(n) / FS
    return x


@pytest.mark.parametrize('estimator', ['allan', 'oallan'])
def test_against_the_oracle_on_device_curves(eng, estimator):
    S, n = 24, 200000
    x = eng.to_device(_series(2, S, n))        # every series' support clear of ties by >= 1.7e-8 of sum w
    var, _ = getattr(eng, estimator)(FS, x, n, S)
    got = _fit(eng, n, var)
    _check(got, var.cpu().numpy(), n, FS, estimator)


def test_against_the_oracle_on_fused_curves(eng):
    from gnss_ins_sim_b200 import imu_model
    n = 120000
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    z = eng.to_device(np.zeros((n, 3)))
    # [5, 6, ntau], read in place; seed 7: every curve's support clear of ties
    avar, _ = eng.allan_mc(FS, 5, z, z, imu.gyro_err, imu.accel_err, 7)
    got = _fit(eng, n, avar)
    assert got.shape == (30, 6)
    _check(got, avar.cpu().numpy().reshape(30, -1), n, FS, 'allan_mc')


def test_every_addressing_gives_the_same_bits(eng):
    S, n = 9, 100000
    xh = _series(2, S, n)
    var, _ = eng.allan(FS, eng.to_device(xh), n, S)
    plain = _fit(eng, n, var)
    ntau = var.shape[1]
    t = var.t().contiguous()                                   # [ntau, S]: series_stride 1, bin_stride S
    assert np.array_equal(_fit(eng, n, t, series_stride=1, bin_stride=S), plain)
    pad = torch.full((S, ntau + 5), float('nan'), dtype=torch.float64, device='cuda')
    pad[:, :ntau] = var                                        # padded rows: series_stride ntau + 5
    assert np.array_equal(_fit(eng, n, pad, series_stride=ntau + 5, nseries=S), plain)
    # K4 on the interleaved [R, n, 3] layout (the reference's per-run arrays) gives the same curves and outputs
    xi = eng.to_device(np.ascontiguousarray(xh.reshape(3, 3, n).transpose(0, 2, 1)))
    vi, _ = eng.allan(FS, xi, n, S, inner=3, outer_stride=3 * n, sample_stride=3)
    assert np.array_equal(_fit(eng, n, vi), plain)
    with pytest.raises(ValueError):
        eng.allan_fit(FS, n, var, series_stride=ntau + 1)


def test_same_bits_whatever_the_batch_and_position(eng):
    S, n = 37, 60000
    var, _ = eng.allan(FS, eng.to_device(_series(3, S, n)), n, S)
    ref = _fit(eng, n, var)
    for s in (0, 5, 36):
        assert np.array_equal(_fit(eng, n, var[s:s + 1].contiguous()), ref[s:s + 1])
    big = var.repeat(29, 1)                                    # 1073 curves: series s at 37 positions
    got = _fit(eng, n, big)
    for rep in range(29):
        assert np.array_equal(got[rep * S:(rep + 1) * S], ref)
    assert np.array_equal(_fit(eng, n, var[4:21].contiguous()), ref[4:21])


@pytest.mark.parametrize('mask', af.SUPPORTS)
def test_model_curves_of_every_support(eng, mask):
    rng = np.random.default_rng(mask)
    base = np.array([1e-8, 1e-6, 1e-8, 1e-10, 1e-13])
    C = np.array([base[i] * 10.0 ** rng.uniform(-0.3, 0.3) if mask >> i & 1 else 0.0 for i in range(5)])
    v = af.model_curve(C, N, FS)
    got = _fit(eng, N, eng.to_device(v[None]))
    _check(got, v[None], N, FS, 'model %d' % mask, need_clear=False)
    Cg = _coef(got[0])
    assert np.all(Cg[C == 0.0] == 0.0) and np.all(np.abs(Cg[C > 0] - C[C > 0]) <= 1e-9 * C[C > 0])


def test_edge_rules(eng):
    base = np.array([1e-8, 1e-6, 1e-8, 1e-10, 1e-13])
    v = af.model_curve(base, N, FS) * np.exp(0.2 * np.random.default_rng(4).standard_normal(len(af.grid(N, FS)[0])))
    ntau = v.size
    rows = [v]
    for bad in (np.nan, np.inf, -np.inf, -1e-9):
        for k in (0, 33, ntau - 1):
            w = v.copy()
            w[k] = bad
            rows.append(w)
    w = v.copy()
    w[3] = 0.0
    rows.append(w)                                             # a zero bin
    rows.append(np.zeros(ntau))                                # all zero
    w = np.zeros(ntau)
    w[[4, 20]] = v[[4, 20]]
    rows.append(w)                                             # two usable bins
    w = np.zeros(ntau)
    w[10] = 2.5e-7
    rows.append(w)                                             # one
    var = np.stack(rows)
    got = _fit(eng, N, eng.to_device(var))
    _check(got, var, N, FS, 'edges', need_clear=False)
    assert np.all(np.isnan(got[1:13]))
    assert got[13][5] == 0.0 and np.all(np.isfinite(got[13]))
    assert np.array_equal(got[14], np.zeros(6))
    # ntau = 0 (80 samples at 10 Hz): six NaNs per series; no series: an empty result
    e = eng.allan_fit(10.0, 80, torch.zeros((3, 0), dtype=torch.float64, device='cuda'))
    assert e.shape == (3, 6) and torch.isnan(e).all()
    assert eng.allan_fit(FS, N, torch.zeros((0, ntau), dtype=torch.float64, device='cuda')).shape == (0, 6)


def _noise(sim, R, which, algo='algo0'):
    d = sim.get_data([which])[0]
    return np.stack([d['%s_%d' % (algo, r)] for r in range(R)])


def _static(n):
    z = np.zeros((n, 3))
    return {'ref_pos': z, 'ref_vel': z, 'ref_att': z, 'ref_accel': np.tile([0.0, 0.0, -9.8], (n, 1)), 'ref_gyro': z}


def _imu(gyro_arw, accel_vrw, gyro_stab=0.0, corr=None):
    from gnss_ins_sim_b200 import imu_model
    z = np.zeros(3)
    acc = {'gyro_b': z, 'gyro_b_stability': np.full(3, gyro_stab), 'gyro_arw': np.full(3, gyro_arw),
           'accel_b': z, 'accel_b_stability': z, 'accel_vrw': np.full(3, accel_vrw)}
    if corr is not None:
        acc['gyro_b_corr'] = np.full(3, corr)
    return imu_model.IMU(accuracy=acc, axis=6, gps=False)


def test_white_noise_law_through_sim(eng):
    """N against the IMU model's arw and vrw (fused K1+K4 path), inside the oracle's white-noise envelope."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    R = 12
    imu = _imu(0.5, 0.05)
    sim = Sim([af.LAW_FS, 0.0, 0.0], _static(af.LAW_N), ref_frame=1, imu=imu, algorithm=Allan(fit=True), seed=5)
    sim.run(R)
    for which, rw in (('noise_gyro', imu.gyro_err['arw']), ('noise_accel', imu.accel_err['vrw'])):
        ratio = _noise(sim, R, which)[:, :, 1] / rw
        ok, got = af.law_check('white', ratio)
        assert ok, (which, got)


def test_rate_random_walk_law_through_sim(eng):
    """A Gauss-Markov drift with b_corr = 1e6 s is a random walk over the hour: K against b_drift sqrt(2 / b_corr),
    inside the oracle's envelope (its white level, N = 1e-4 rad/s/sqrt(Hz), and K = 3e-5 are the law case's)."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    R, corr = 12, 1e6
    K = af.LAWS['rw']['truth']
    drift = K / np.sqrt(2.0 / corr)                            # rad/s
    imu = _imu(1e-4 * 60.0 / np.pi * 180.0, 0.0, gyro_stab=drift * 180.0 / np.pi * 3600.0, corr=corr)
    assert np.allclose(imu.gyro_err['arw'], 1e-4) and np.allclose(imu.gyro_err['b_drift'], drift)
    sim = Sim([af.LAW_FS, 0.0, 0.0], _static(af.LAW_N), ref_frame=1, imu=imu, algorithm=Allan(fit=True), seed=8)
    sim.run(R)
    ratio = _noise(sim, R, 'noise_gyro')[:, :, 3] / K
    ok, got = af.law_check('rw', ratio)
    assert ok, got


def _logged(path, kind, R, seed):
    rng = np.random.default_rng(seed)
    n = af.LAW_N
    os.makedirs(path, exist_ok=True)
    np.savetxt(os.path.join(path, 'time.csv'), np.arange(n) / af.LAW_FS, header='time (sec)', comments='')
    for r in range(R):
        g = np.stack([af.law_series(kind, rng) for _ in range(3)], axis=1)
        np.savetxt(os.path.join(path, 'gyro-%d.csv' % r), g, delimiter=',', comments='', fmt='%.17e',
                   header='gyro_x (rad/s),gyro_y (rad/s),gyro_z (rad/s)')
        np.savetxt(os.path.join(path, 'accel-%d.csv' % r), g + np.array([0.0, 0.0, -9.8]), delimiter=',',
                   comments='', fmt='%.17e', header='accel_x (m/s^2),accel_y (m/s^2),accel_z (m/s^2)')
    return path


@pytest.mark.parametrize('kind', ['ramp', 'quant'])
def test_ramp_and_quantisation_laws_from_logged_directories(eng, tmp_path, kind):
    """A logged directory of white noise plus a rate ramp (R), or of a quantised angle, differenced (Q): inside the
    oracle's envelopes, and the plugin on the same arrays gives the same bits."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    R = 4
    d = _logged(str(tmp_path / kind), kind, R, 50 + len(kind))
    sim = Sim([af.LAW_FS, 0.0, 0.0], d, ref_frame=0, imu=None, algorithm=Allan(fit=True))
    sim.run(R)
    c = af.LAWS[kind]
    ng, na = _noise(sim, R, 'noise_gyro'), _noise(sim, R, 'noise_accel')
    ok, got = af.law_check(kind, ng[:, :, c['col']] / c['truth'])
    assert ok, got
    sets = [np.genfromtxt(os.path.join(d, 'gyro-%d.csv' % r), delimiter=',', skip_header=1) for r in range(R)]
    acc = [np.genfromtxt(os.path.join(d, 'accel-%d.csv' % r), delimiter=',', skip_header=1) for r in range(R)]
    _, _, _, pa, pg = Allan(fit=True).run_batch(af.LAW_FS, np.stack(acc), np.stack(sets))
    assert np.array_equal(pg, ng) and np.array_equal(pa, na)


def test_sim_paths_agree_with_engine_and_save_data(eng, monkeypatch, tmp_path):
    """The fused and the materialised Sim paths give engine.allan_fit of the same curves bit for bit; a vibration
    environment's path fits its own curves; Allan(fit=False) publishes no noise_*; save_data writes noise_*."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    from gnss_ins_sim_b200 import imu_model
    n, R, seed = 60000, 5, 21
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    traj = _static(n)
    rg, ra = eng.to_device(traj['ref_gyro']), eng.to_device(traj['ref_accel'])
    sim = Sim([FS, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Allan(fit=True), seed=seed)
    sim.run(R)
    avar, _ = eng.allan_mc(FS, R, rg, ra, imu.gyro_err, imu.accel_err, seed)
    want = eng.allan_fit(FS, n, avar).reshape(R, 6, 6).cpu().numpy()
    na, ng = _noise(sim, R, 'noise_accel'), _noise(sim, R, 'noise_gyro')
    assert np.array_equal(na, want[:, 0:3]) and np.array_equal(ng, want[:, 3:6])
    plain = Sim([FS, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Allan(), seed=seed)
    plain.run(R)
    assert 'noise_gyro' not in plain.data
    assert all(np.array_equal(plain.data['ad_gyro'][k], sim.data['ad_gyro'][k]) for k in sim.data['ad_gyro'])
    # materialised (K1 then K4), in small run blocks
    monkeypatch.setenv('B2INS_ALLAN_FUSED', '0')
    monkeypatch.setattr(Sim, '_allan_block', lambda self, *a: 2)
    for overlapping in (False, True):
        sm = Sim([FS, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Allan(overlapping, fit=True), seed=seed)
        sm.run(R)
        gyro, accel = eng.imu_noise(FS, R, rg, ra, imu.gyro_err, imu.accel_err, seed,
                                    layout=eng.LAYOUT_CHANNEL_MAJOR)
        est = eng.oallan if overlapping else eng.allan
        for x, which in ((accel, 'noise_accel'), (gyro, 'noise_gyro')):
            v, _ = est(FS, x, n, 3 * R)
            assert np.array_equal(_noise(sm, R, which), eng.allan_fit(FS, n, v).reshape(R, 3, 6).cpu().numpy())
    monkeypatch.delenv('B2INS_ALLAN_FUSED')
    # a vibration environment (materialised with its vibration): the fit of its own published curves
    sv = Sim([FS, 0.0, 0.0], traj, ref_frame=1, imu=imu, env={'acc': '[0.1 0.1 0.1]-random'},
             algorithm=Allan(fit=True), seed=seed)
    sv.run(R)
    for which, dev in (('noise_accel', 'ad_accel'), ('noise_gyro', 'ad_gyro')):
        ad = np.stack([sv.data[dev]['algo0_%d' % r] for r in range(R)])          # [R, ntau, 3]
        v = eng.to_device(np.ascontiguousarray((ad * ad).transpose(0, 2, 1)))
        ref = eng.allan_fit(FS, n, v).reshape(R, 3, 6).cpu().numpy()
        got = _noise(sv, R, which)
        assert np.all(np.abs(got - ref) <= 1e-9 * np.abs(ref)), which
    # save_data: one row per axis, the units in the header, the values as they are
    out = str(tmp_path / 'out')
    sim.save_data(out, names=['noise_gyro', 'noise_accel'])
    back = np.genfromtxt(os.path.join(out, 'noise_gyro-algo0_3.csv'), delimiter=',', skip_header=1)
    assert np.array_equal(back, ng[3])
    with open(os.path.join(out, 'noise_accel-algo0_0.csv')) as fp:
        assert fp.readline().strip() == ('Q (m/s),N (m/s^2/sqrt(Hz)),B (m/s^2),K (m/s^3/sqrt(Hz)),R (m/s^3),'
                                         'B_min (m/s^2)')


def _two_rank_worker(rank, world, port, tmp):
    """One rank of a two-rank Sim (a gloo group; both ranks on the first GPU): Allan(fit=True) on the fused and
    on the materialised path, its 5 runs sharded 3 + 2."""
    import sys
    import torch.distributed as td
    from conftest import ROOT
    sys.path.insert(0, ROOT)
    torch.cuda.set_device(0)
    td.init_process_group('gloo', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world)
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    out = {}
    for overlapping in (False, True):
        sim = Sim([FS, 0.0, 0.0], _static(30000), ref_frame=1, imu=imu, algorithm=Allan(overlapping, fit=True),
                  seed=7)
        sim.run(5)
        for which in ('noise_accel', 'noise_gyro', 'ad_gyro'):
            out['%s_%d' % (which, overlapping)] = _noise(sim, 5, which)
        out['local_%d' % overlapping] = sim._shard[1] - sim._shard[0]
    np.savez(os.path.join(tmp, 'r%d.npz' % rank), **out)
    td.destroy_process_group()


def test_two_ranks_gather_the_noise_terms(eng, tmp_path):
    """Two ranks, each fitting its shard of the runs, publish the same noise terms and curves as one process."""
    import socket
    import torch.multiprocessing as mp
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    with socket.socket() as sk:
        sk.bind(('127.0.0.1', 0))
        port = sk.getsockname()[1]
    mp.spawn(_two_rank_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    for overlapping in (False, True):
        one = Sim([FS, 0.0, 0.0], _static(30000), ref_frame=1, imu=imu, algorithm=Allan(overlapping, fit=True), seed=7)
        one.run(5)
        locals_ = []
        for r in range(2):
            z = np.load(os.path.join(str(tmp_path), 'r%d.npz' % r))
            for which in ('noise_accel', 'noise_gyro', 'ad_gyro'):
                assert np.array_equal(z['%s_%d' % (which, overlapping)], _noise(one, 5, which)), (r, which)
            locals_.append(int(z['local_%d' % overlapping]))
        assert sorted(locals_) == [2, 3]
