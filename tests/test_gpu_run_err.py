"""Run-to-run bias, scale-factor and misalignment errors on the GPU: the run-error table and K1's and K9's _rx forms
held to oracle/run_err_np.py, the zero-error dispatch, the yaw laws of a scale factor and a turn-on bias through
Sim, and the consumers that take the errors through K1 (free integration, Allan, Psd)."""
import ctypes

import numpy as np
import pytest

import run_err_np as rx
from conftest import assert_close, load_golden, wrap_pi

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

FS = 100.0
SEED = 41
MA_G = np.array([[0.0, 2e-3, 1e-3], [3e-3, 0.0, 4e-3], [5e-4, 6e-3, 0.0]])
RUN = ({'b_std': np.array([1e-4, 2e-4, 5e-5]), 'sf': np.array([1e-3, 2e-3, 5e-4]), 'ma': MA_G},
       {'b_std': np.array([1e-2, 3e-2, 2e-2]), 'sf': np.array([3e-3, 1e-3, 2e-3]), 'ma': 2e-3 * (1.0 - np.eye(3))})
TERMS = ({'q': np.array([2e-5, 1e-5, 3e-5]), 'rrw': np.array([3e-5, 1e-5, 5e-5]), 'rr': np.array([1e-6, -2e-6, 3e-7])},
         {'q': np.array([1e-3, 2e-3, 5e-4]), 'rrw': np.array([1e-3, 3e-4, 2e-3]), 'rr': np.array([1e-4, 0.0, -2e-4])})


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _errs(run=True, terms=False):
    g = {'b': np.array([1e-4, 0.0, -2e-4]), 'b_drift': np.full(3, 1e-5), 'b_corr': np.array([100.0, np.inf, 5.0]),
         'arw': np.full(3, 1e-4)}
    a = {'b': np.array([0.01, 0.0, -0.02]), 'b_drift': np.full(3, 1e-3), 'b_corr': np.array([np.inf, 50.0, 1.0]),
         'vrw': np.full(3, 1e-3)}
    for s, d in enumerate((a, g)):
        if run:
            d.update(RUN[1 - s])
        if terms:
            d.update(TERMS[1 - s])
    return g, a


def _ref(n, seed=5):
    rng = np.random.default_rng(seed)
    return 0.1 * rng.standard_normal((n, 3)), np.array([0.0, 0.0, -9.8]) + 0.1 * rng.standard_normal((n, 3))


def _run_major(eng, x, layout):
    if layout == eng.LAYOUT_TIME_MAJOR:
        return x.permute(2, 0, 1)
    if layout == eng.LAYOUT_CHANNEL_MAJOR:
        return x.permute(0, 2, 1)
    return x


def _table(ge, ae, seed, runs):
    return np.stack([rx.table(ae, 0, seed, runs), rx.table(ge, 1, seed, runs)], axis=1)


def _sigma(ge, ae):
    """[2, 3, 4] the 1-sigma value of every table entry (accel, gyro; S, then b_run)."""
    out = np.zeros((2, 3, 4))
    for s, err in enumerate((ae, ge)):
        b, sf, ma = rx.sigmas(err)
        out[s, :, :3] = ma + np.diag(sf)
        out[s, :, 3] = b
    return out


@pytest.mark.parametrize('r0', [0, 5, 2 ** 32 - 3, 2 ** 32 - 1])
def test_run_error_table_matches_the_oracle(eng, r0):
    """engine.imu_run_errors against run_err_np.table to 1e-13 of each entry's sigma (the device/NumPy agreement of
    the unit normals, tests/test_gpu_parity.py); the same bits for any block split of the runs."""
    ge, ae = _errs()
    R = 10
    got = eng.imu_run_errors(R, ge, ae, SEED, run_offset=r0).cpu().numpy()
    want = _table(ge, ae, SEED, np.arange(r0, r0 + R, dtype=np.uint64))
    assert got.shape == (R, 2, 3, 4)
    sigma = _sigma(ge, ae)
    assert np.all(np.abs(got - want) <= 1e-13 * sigma), np.max(np.abs(got - want) / np.where(sigma > 0, sigma, 1))
    assert np.all((got == 0.0) == (want == 0.0))
    parts = [eng.imu_run_errors(k1 - k0, ge, ae, SEED, run_offset=r0 + k0).cpu().numpy()
             for k0, k1 in ((0, 3), (3, 4), (4, 10))]
    assert np.array_equal(np.concatenate(parts), got)
    # an IMU without run errors: a zero table
    g0, a0 = _errs(run=False)
    assert not np.any(eng.imu_run_errors(3, g0, a0, SEED).cpu().numpy())


@pytest.mark.parametrize('terms', [False, True])
@pytest.mark.parametrize('layout', [0, 1, 2])
def test_k1_rx_matches_the_oracle(eng, terms, layout):
    for R, n, r0 in ((5, 897, 3), (3, 1793, 2 ** 32 - 1)):
        rg, ra = _ref(n)
        ge, ae = _errs(terms=terms)
        g, a = eng.imu_noise(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=r0,
                             layout=layout)
        og, oa = rx.imu_noise(FS, rg, ra, ge, ae, SEED, np.arange(r0, r0 + R, dtype=np.uint64))
        assert_close(_run_major(eng, g, layout).cpu().numpy(), og, 1e-12, 1.0, 'gyro')
        assert_close(_run_major(eng, a, layout).cpu().numpy(), oa, 1e-12, 1.0, 'accel')


@pytest.mark.parametrize('vib', ['random', 'sinusoidal'])
def test_k1_rx_with_vibration(eng, vib):
    """The vibration is an error term: M = I + S scales the truth, not the vibration."""
    R, n = 4, 1000
    rg, ra = _ref(n)
    ge, ae = _errs(terms=True)
    va = {'type': vib, 'x': 0.01, 'y': 0.02, 'z': 0.03, 'freq': 7.0}
    vg = {'type': vib, 'x': 1e-3, 'y': 2e-3, 'z': 3e-3, 'freq': 11.0}
    g, a = eng.imu_noise(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=1, vib_gyro=vg,
                         vib_accel=va)
    og, oa = rx.imu_noise(FS, rg, ra, ge, ae, SEED, np.arange(1, 1 + R), vib_acc=va, vib_gyro=vg)
    assert_close(g.cpu().numpy(), og, 1e-12, 1.0, 'gyro')
    assert_close(a.cpu().numpy(), oa, 1e-12, 1.0, 'accel')


def _check_proc(proc, e):
    assert_close(proc[:, 0], np.max(np.abs(e), 1), 1e-12, 1.0, 'max')
    assert_close(proc[:, 1], np.mean(e, 1), 1e-10, 1e-3, 'mean')
    assert_close(proc[:, 2], np.std(e, 1), 1e-10, 1e-3, 'std')


@pytest.mark.parametrize('terms', [False, True])
def test_k1_rx_time_segments(eng, terms):
    """Two runs of 2^18 + 1001 samples take the segmented plan: every segment's CTA draws the same run errors."""
    from gnss_ins_sim_b200 import _lib
    R, n = 2, (1 << 18) + 1001
    rg, ra = _ref(n, 9)
    ge, ae = _errs(terms=terms)
    assert _lib.noise_plan(FS, R, n, ge, ae)['nseg'] > 1
    g, a = eng.imu_noise(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=7)
    og, oa = rx.imu_noise(FS, rg, ra, ge, ae, SEED, np.arange(7, 7 + R))
    assert_close(g.cpu().numpy(), og, 1e-12, 1.0, 'gyro')
    assert_close(a.cpu().numpy(), oa, 1e-12, 1.0, 'accel')
    end, proc = eng.imu_err_stats(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=7,
                                  stats_start=12345)
    e = np.concatenate([oa - ra[None], og - rg[None]], axis=2)
    assert_close(end.cpu().numpy(), e[:, -1], 1e-12, 1.0, 'end')
    _check_proc(proc.cpu().numpy(), e[:, 12345:])


@pytest.mark.parametrize('terms', [False, True])
@pytest.mark.parametrize('start', [-1, 0, 333])
def test_k9_rx_matches_the_oracle_statistics(eng, terms, start):
    R, n = 6, 2500
    rg, ra = _ref(n)
    ge, ae = _errs(terms=terms)
    end, proc = eng.imu_err_stats(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=4,
                                  stats_start=start)
    og, oa = rx.imu_noise(FS, rg, ra, ge, ae, SEED, np.arange(4, 4 + R))
    e = np.concatenate([oa - ra[None], og - rg[None]], axis=2)
    assert_close(end.cpu().numpy(), e[:, -1], 1e-12, 1.0, 'end')
    if start >= 0:
        _check_proc(proc.cpu().numpy(), e[:, start:])
    else:
        assert proc is None


def test_run_errors_disturb_no_other_draw(eng):
    """K1-rx minus K1-ex of the same IMU without the run-error keys is delta = b_run + S ref, computed on the host
    from the device's own table: the new draws leave every other stream as it was."""
    R, n = 5, 3000
    rg, ra = _ref(n)
    ge, ae = _errs(terms=True)
    g0, a0 = _errs(run=False, terms=True)
    drg, dra = eng.to_device(rg), eng.to_device(ra)
    g1, a1 = eng.imu_noise(FS, R, drg, dra, ge, ae, SEED, run_offset=11)
    g2, a2 = eng.imu_noise(FS, R, drg, dra, g0, a0, SEED, run_offset=11)
    tab = eng.imu_run_errors(R, ge, ae, SEED, run_offset=11).cpu().numpy()
    for name, x, y, sensor, ref in (('gyro', g1, g2, 1, rg), ('accel', a1, a2, 0, ra)):
        d = rx.delta(ref, tab[:, sensor])
        assert_close((x - y).cpu().numpy(), d, 1e-12, np.abs(y.cpu().numpy()).max(), name)


def test_zero_run_errors_through_the_rx_entry_points_are_the_plain_ones(eng):
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    R, n = 3, 2000
    rg, ra = _ref(n)
    drg, dra = eng.to_device(rg), eng.to_device(ra)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    zero = _lib.RunErr()
    for terms in (False, True):
        ge, ae = _errs(run=False, terms=terms)
        g0, a0 = eng.imu_noise(FS, R, drg, dra, ge, ae, SEED, run_offset=2)       # plain or _ex
        e0, p0 = eng.imu_err_stats(FS, R, drg, dra, ge, ae, SEED, run_offset=2, stats_start=100)
        se_g, se_a, vib = _lib.sensor_err(ge, 'arw'), _lib.sensor_err(ae, 'vrw'), _lib.vib(None)
        tg, ta = _lib.noise_terms(ge), _lib.noise_terms(ae)
        for xg, xa in ((None, None), (ctypes.byref(zero), ctypes.byref(zero))):
            g1, a1 = torch.empty_like(g0), torch.empty_like(a0)
            _lib.check(lib.b2ins_imu_noise_rx_f64(FS, R, n, p(drg), p(dra), ctypes.byref(se_g), ctypes.byref(se_a),
                                                  tg, ta, ctypes.byref(vib), ctypes.byref(vib), SEED, 2, 0, p(g1),
                                                  p(a1), None, xg, xa, None))
            e1, p1 = torch.empty_like(e0), torch.empty_like(p0)
            _lib.check(lib.b2ins_imu_err_stats_rx_f64(FS, R, n, p(drg), p(dra), ctypes.byref(se_g),
                                                      ctypes.byref(se_a), tg, ta, ctypes.byref(vib),
                                                      ctypes.byref(vib), SEED, 2, 100, p(e1), p(p1), xg, xa, None))
            torch.cuda.synchronize()
            assert torch.equal(g0, g1) and torch.equal(a0, a1), terms
            assert torch.equal(e0, e1) and torch.equal(p0, p1), terms
        # the dict path: keys present but zero take the same kernels
        gz, az = dict(ge, b_std=np.zeros(3), sf=np.zeros(3), ma=np.zeros((3, 3))), dict(ae, sf=0.0)
        g2, a2 = eng.imu_noise(FS, R, drg, dra, gz, az, SEED, run_offset=2)
        assert torch.equal(g0, g2) and torch.equal(a0, a2)


# ---- the yaw laws through Sim: a scale factor and a turn-on bias on the 90-degree turn ----------------------------
def _turn_sim(acc, runs, force=False):
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    g = load_golden('traj_90deg_turn_100hz_rf1.npz')
    traj = {k: g[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    zero = {'gyro_b': [0.0] * 3, 'gyro_b_stability': [0.0] * 3, 'gyro_arw': [0.0] * 3,
            'accel_b': [0.0] * 3, 'accel_b_stability': [0.0] * 3, 'accel_vrw': [0.0] * 3}
    imu = imu_model.IMU(dict(zero, **acc), gps=False)
    sim = Sim([100.0, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=FreeIntegration(g['ini']), seed=SEED,
              run_base=1000)
    sim._force_fed = force
    sim.run(runs)
    return sim, g


@pytest.mark.parametrize('kind', ['sf', 'b_std'])
def test_yaw_laws_of_the_run_errors(eng, kind):
    """ref_frame 1 integrates yaw by forward Euler, att[i] = att[i-1] + w[i-1] dt (i = 1 .. n-1, mech.cuh as
    free_integration.py:104), and roll and pitch stay 0 on this trajectory (ref_gyro x, y are 0 and so are the
    errors there): the end yaw is linear in gyro z.  Over 1000 runs, the end yaw error minus that of an error-free
    IMU on the same route is sf_z sum_{i<n-1} ref_gyro_z[i] dt (about sf_z pi/2), or b_run_z (n - 1) dt."""
    R = 1000
    acc = {'gyro_sf': [0.0, 0.0, 1000.0]} if kind == 'sf' else {'gyro_b_std': [0.0, 0.0, 36.0]}
    sim, g = _turn_sim(acc, R)
    base, _ = _turn_sim({}, 1, force=True)
    tab = sim.imu_run_errors()['gyro']
    assert tab.shape == (R, 3, 4)
    n, dt = g['ref_gyro'].shape[0], 1.0 / 100.0
    if kind == 'sf':
        coef = tab[:, 2, 2]
        want = coef * (np.sum(g['ref_gyro'][:n - 1, 2]) * dt)
        np.testing.assert_allclose(np.sum(g['ref_gyro'][:n - 1, 2]) * dt, np.pi / 2, rtol=1e-12)
    else:
        coef = tab[:, 2, 3]
        want = coef * ((n - 1) * dt)
    assert np.count_nonzero(tab) == R            # only the one parameter is drawn non-zero
    assert np.std(coef) > 0.5 * (1e-3 if kind == 'sf' else 36.0 * np.pi / 180.0 / 3600.0)
    end, end0 = sim.end_point_errors(), base.end_point_errors()
    dyaw = wrap_pi(end[:, 0] - end0[0, 0])
    assert np.max(np.abs(dyaw - want)) <= 1e-12, np.max(np.abs(dyaw - want))
    assert np.max(np.abs(end[:, 1:3])) <= 1e-12          # pitch and roll
    # the table is drawn from the global run ids run_base + r
    t7 = eng.imu_run_errors(5, sim.imu.gyro_err, sim.imu.accel_err, SEED, run_offset=1007).cpu().numpy()
    assert np.array_equal(t7[:, 1], tab[7:12])


# ---- the consumers: free integration, Allan and Psd on K1-rx's series ---------------------------------------------
@pytest.mark.parametrize('rf', [1, 0])
def test_free_integration_with_run_errors_is_k2_on_k1_rx(eng, rf):
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    from gnss_ins_sim_b200.allan_analysis import Allan
    from gnss_ins_sim_b200.psd_analysis import Psd
    acc = {'gyro_b': [0.0] * 3, 'gyro_b_stability': [3.5] * 3, 'gyro_arw': [0.25] * 3, 'gyro_b_corr': [100.0] * 3,
           'accel_b': [0.0] * 3, 'accel_b_stability': [5e-5] * 3, 'accel_vrw': [0.03] * 3,
           'accel_b_corr': [100.0] * 3, 'gyro_b_std': [10.0] * 3, 'gyro_sf': [500.0, 800.0, 1000.0],
           'gyro_ma': 0.05, 'accel_b_std': [0.01] * 3, 'accel_sf': [300.0] * 3, 'accel_ma': 0.02}
    imu = imu_model.IMU(acc, gps=False)
    g = load_golden('philox_90deg_mid_rf%d.npz' % rf)
    traj = {k: g[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    seed = int(g['seed'])
    sim = Sim([100.0, 0.0, 0.0], traj, ref_frame=rf, imu=imu, algorithm=FreeIntegration(g['ini']), seed=seed)
    R = 6
    sim.run(R)
    dev = eng.to_device
    gyro, accel = eng.imu_noise(100.0, R, dev(g['ref_gyro']), dev(g['ref_accel']), imu.gyro_err, imu.accel_err, seed)
    att, pos, vel = eng.free_integration(rf, 100.0, gyro, accel, dev(np.asarray(g['ini'])[None]))
    att, pos, vel = (t.cpu().numpy() for t in (att, pos, vel))
    end = np.concatenate([wrap_pi(att[:, -1] - g['ref_att'][-1]), pos[:, -1] - g['ref_pos'][-1],
                          vel[:, -1] - g['ref_vel'][-1]], axis=1)
    scale = lambda x: max(1.0, np.max(np.abs(x)))  # noqa: E731
    got = sim.end_point_errors()
    assert np.max(np.abs(got - end)) <= 1e-12 * scale(end)
    st = sim.get_error_stats('vel', -1)
    assert np.max(np.abs(st['std'] - np.std(end[:, 6:9], 0))) <= 1e-9 * scale(end[:, 6:9])
    ps = sim.get_error_stats('pos', 2.5)
    e = pos[:, 250:] - g['ref_pos'][None, 250:]
    avg = np.stack([ps['avg']['algo0_%d' % r] for r in range(R)])
    assert np.max(np.abs(avg - e.mean(1))) <= 1e-12 * scale(e)
    assert np.array_equal(sim.get_data(['accel'])[0][2], accel[2].cpu().numpy())
    # the run errors reach the sensor statistics (K9-rx)
    sg = sim.get_error_stats('gyro', -1)
    want = (gyro.cpu().numpy()[:, -1] - g['ref_gyro'][-1]).mean(0)
    assert np.max(np.abs(sg['avg'] - want)) <= 1e-12 * scale(want)
    # Allan and Psd through Sim run the materialised path on K1-rx's series
    s2 = Sim([100.0, 0.0, 0.0], traj, ref_frame=rf, imu=imu, algorithm=Allan(), seed=seed)
    s2.run(R)
    gc = gyro.permute(0, 2, 1).contiguous()
    v, _ = eng.allan(100.0, gc, gc.shape[2], R * 3)
    ad = np.sqrt(v.cpu().numpy()).reshape(R, 3, -1).transpose(0, 2, 1)
    got = np.stack([s2.get_data(['ad_gyro'])[0]['algo0_%d' % r] for r in range(R)])
    assert np.max(np.abs(got - ad)) <= 1e-12 * np.max(ad)
    s3 = Sim([100.0, 0.0, 0.0], traj, ref_frame=rf, imu=imu, algorithm=Psd(nperseg=256), seed=seed)
    s3.run(R)
    gm, am = (eng.imu_noise(100.0, R, dev(g['ref_gyro']), dev(g['ref_accel']), imu.gyro_err, imu.accel_err, seed,
                            layout=eng.LAYOUT_CHANNEL_MAJOR))
    f2, a2, g2 = Psd(nperseg=256).run_batch(100.0, am, gm, channel_major=True)
    pa, pg = (np.stack([s3.get_data([k])[0]['algo0_%d' % r] for r in range(R)]) for k in ('psd_accel', 'psd_gyro'))
    assert np.array_equal(pa, a2) and np.array_equal(pg, g2)
