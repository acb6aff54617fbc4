"""The IEEE Std 952 terms on the GPU: K1's and K9's _ex forms held to oracle/noise952_np.py, the zero-term
dispatch, the Allan and Hadamard laws of the generated ensemble, and free integration through K1 then K2."""
import ctypes
import math

import numpy as np
import pytest

import allan_fit_np as af
import noise952_np as nz
from conftest import assert_close, load_golden, wrap_pi

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

FS = 100.0
SEED = 41
TERMS = {'q': ({'q': np.array([2e-5, 1e-5, 3e-5])}, {'q': np.array([1e-3, 2e-3, 5e-4])}),
         'rrw': ({'rrw': np.array([3e-5, 1e-5, 5e-5])}, {'rrw': np.array([1e-3, 3e-4, 2e-3])}),
         'rr': ({'rr': np.array([1e-6, -2e-6, 3e-7])}, {'rr': np.array([1e-4, 0.0, -2e-4])})}
TERMS['all'] = tuple({k: v for t in TERMS.values() for k, v in t[s].items()} for s in (0, 1))


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _errs(terms='all'):
    g = {'b': np.array([1e-4, 0.0, -2e-4]), 'b_drift': np.full(3, 1e-5), 'b_corr': np.array([100.0, np.inf, 5.0]),
         'arw': np.full(3, 1e-4)}
    a = {'b': np.array([0.01, 0.0, -0.02]), 'b_drift': np.full(3, 1e-3), 'b_corr': np.array([np.inf, 50.0, 1.0]),
         'vrw': np.full(3, 1e-3)}
    if terms:
        g.update(TERMS[terms][0])
        a.update(TERMS[terms][1])
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


@pytest.mark.parametrize('terms', ['q', 'rrw', 'rr', 'all'])
@pytest.mark.parametrize('layout', [0, 1, 2])
def test_k1_ex_matches_the_oracle(eng, terms, layout):
    for R, n, r0 in ((5, 897, 3), (3, 1793, 2 ** 32 - 1)):
        rg, ra = _ref(n)
        ge, ae = _errs(terms)
        g, a = eng.imu_noise(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=r0,
                             layout=layout)
        og, oa = nz.imu_noise(FS, rg, ra, ge, ae, SEED, np.arange(r0, r0 + R, dtype=np.uint64))
        assert_close(_run_major(eng, g, layout).cpu().numpy(), og, 1e-12, 1.0, 'gyro %s' % terms)
        assert_close(_run_major(eng, a, layout).cpu().numpy(), oa, 1e-12, 1.0, 'accel %s' % terms)


@pytest.mark.parametrize('vib', ['random', 'sinusoidal'])
def test_k1_ex_with_vibration(eng, vib):
    R, n = 4, 1000
    rg, ra = _ref(n)
    ge, ae = _errs('all')
    va = {'type': vib, 'x': 0.01, 'y': 0.02, 'z': 0.03, 'freq': 7.0}
    vg = {'type': vib, 'x': 1e-3, 'y': 2e-3, 'z': 3e-3, 'freq': 11.0}
    g, a = eng.imu_noise(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=1, vib_gyro=vg,
                         vib_accel=va)
    og, oa = nz.imu_noise(FS, rg, ra, ge, ae, SEED, np.arange(1, 1 + R), vib_acc=va, vib_gyro=vg)
    assert_close(g.cpu().numpy(), og, 1e-12, 1.0, 'gyro')
    assert_close(a.cpu().numpy(), oa, 1e-12, 1.0, 'accel')


def test_k1_ex_time_segments_carry_the_walk(eng):
    """Two runs of 2^18 + 1001 samples take the segmented plan; the walk never decays, so pass 1 covers whole
    segments, and the walk is carried across the segment ends with a = 1."""
    from gnss_ins_sim_b200 import _lib
    R, n = 2, (1 << 18) + 1001
    rg, ra = np.zeros((n, 3)), np.zeros((n, 3))
    ge, ae = _errs('all')
    plan = _lib.noise_plan(FS, R, n, ge, ae)
    assert plan['nseg'] > 1 and plan['pass1_len'] == plan['seg_len']
    # with short correlation times pass 1 is shortened, unless a rate random walk is set
    short_g, short_a = dict(ge, b_corr=np.full(3, 0.5)), dict(ae, b_corr=np.full(3, 0.5))
    for key, whole in (('rrw', True), ('q', False), ('rr', False)):
        g1 = {k: v for k, v in short_g.items() if k not in ('q', 'rrw', 'rr') or k == key}
        a1 = {k: v for k, v in short_a.items() if k not in ('q', 'rrw', 'rr') or k == key}
        p1 = _lib.noise_plan(FS, R, n, g1, a1)
        assert p1['nseg'] == plan['nseg'] and (p1['pass1_len'] == p1['seg_len']) == whole, key
    g, a = eng.imu_noise(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=7)
    og, oa = nz.imu_noise(FS, rg, ra, ge, ae, SEED, np.arange(7, 7 + R))
    assert_close(g.cpu().numpy(), og, 1e-12, 1.0, 'gyro')
    assert_close(a.cpu().numpy(), oa, 1e-12, 1.0, 'accel')
    # K9-ex on the same plan
    end, proc = eng.imu_err_stats(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=7,
                                  stats_start=12345)
    e = np.concatenate([oa, og], axis=2)
    assert_close(end.cpu().numpy(), e[:, -1], 1e-12, 1.0, 'end')
    _check_proc(proc.cpu().numpy(), e[:, 12345:])


def _check_proc(proc, e):
    assert_close(proc[:, 0], np.max(np.abs(e), 1), 1e-12, 1.0, 'max')
    assert_close(proc[:, 1], np.mean(e, 1), 1e-10, 1e-3, 'mean')
    assert_close(proc[:, 2], np.std(e, 1), 1e-10, 1e-3, 'std')


def test_zero_terms_through_the_ex_entry_points_are_the_plain_ones(eng):
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    R, n = 3, 2000
    rg, ra = _ref(n)
    ge, ae = _errs(None)
    drg, dra = eng.to_device(rg), eng.to_device(ra)
    g0, a0 = eng.imu_noise(FS, R, drg, dra, ge, ae, SEED, run_offset=2)
    e0, p0 = eng.imu_err_stats(FS, R, drg, dra, ge, ae, SEED, run_offset=2, stats_start=100)
    zero = _lib.NoiseTerms()
    se_g, se_a, vib = _lib.sensor_err(ge, 'arw'), _lib.sensor_err(ae, 'vrw'), _lib.vib(None)
    g1, a1 = torch.empty_like(g0), torch.empty_like(a0)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    for tg, ta in ((None, None), (ctypes.byref(zero), ctypes.byref(zero))):
        _lib.check(lib.b2ins_imu_noise_ex_f64(FS, R, n, p(drg), p(dra), ctypes.byref(se_g), ctypes.byref(se_a), tg,
                                              ta, ctypes.byref(vib), ctypes.byref(vib), SEED, 2, 0, p(g1), p(a1),
                                              None, None))
        e1, p1 = torch.empty_like(e0), torch.empty_like(p0)
        _lib.check(lib.b2ins_imu_err_stats_ex_f64(FS, R, n, p(drg), p(dra), ctypes.byref(se_g), ctypes.byref(se_a),
                                                  tg, ta, ctypes.byref(vib), ctypes.byref(vib), SEED, 2, 100, p(e1),
                                                  p(p1), None))
        torch.cuda.synchronize()
        assert torch.equal(g0, g1) and torch.equal(a0, a1)
        assert torch.equal(e0, e1) and torch.equal(p0, p1)
    # the dict path: keys present but zero take the plain kernels too
    gz, az = _errs(None)
    gz.update(q=np.zeros(3), rrw=np.zeros(3), rr=np.zeros(3))
    g2, a2 = eng.imu_noise(FS, R, drg, dra, gz, az, SEED, run_offset=2)
    assert torch.equal(g0, g2) and torch.equal(a0, a2)
    # bad terms are refused before any launch
    bad = _lib.NoiseTerms()
    bad.k[1] = -1.0
    with pytest.raises(ValueError, match='noise terms'):
        _lib.check(lib.b2ins_imu_noise_ex_f64(FS, R, n, p(drg), p(dra), ctypes.byref(se_g), ctypes.byref(se_a),
                                              ctypes.byref(bad), None, ctypes.byref(vib), ctypes.byref(vib), SEED, 2,
                                              0, p(g1), p(a1), None, None))


@pytest.mark.parametrize('start', [-1, 0, 333])
def test_k9_ex_matches_the_oracle_statistics(eng, start):
    R, n = 6, 2500
    rg, ra = _ref(n)
    ge, ae = _errs('all')
    end, proc = eng.imu_err_stats(FS, R, eng.to_device(rg), eng.to_device(ra), ge, ae, SEED, run_offset=4,
                                  stats_start=start)
    og, oa = nz.imu_noise(FS, rg, ra, ge, ae, SEED, np.arange(4, 4 + R))
    e = np.concatenate([oa - ra[None], og - rg[None]], axis=2)
    assert_close(end.cpu().numpy(), e[:, -1], 1e-12, 1.0, 'end')
    if start >= 0:
        _check_proc(proc.cpu().numpy(), e[:, start:])
    else:
        assert proc is None


@pytest.mark.parametrize('case', ['white+quant', 'white+rrw', 'white+ramp', 'all'])
def test_laws_of_the_generated_ensemble(eng, case):
    """Over 2000 runs the ensemble mean of K4, K4o and the overlapping Hadamard variance at every tau agrees with
    the closed forms (noise952_np) within 5 standard errors of the ensemble; the ramp leaves the Hadamard curve."""
    R, n, dt = 2000, 3000, 1.0 / FS
    p = {'N': 1e-4}
    terms = {}
    if case in ('white+quant', 'all'):
        p['Q'], terms['q'] = 3e-5, np.full(3, 3e-5)
    if case in ('white+rrw', 'all'):
        p['K'], terms['rrw'] = 2e-4, np.full(3, 2e-4)
    if case in ('white+ramp', 'all'):
        p['R'], terms['rr'] = 1e-4, np.full(3, 1e-4)
    err = dict({'b': np.full(3, 0.3), 'b_drift': np.zeros(3), 'b_corr': np.full(3, np.inf), 'arw': np.full(3, p['N'])},
               **terms)
    ref = eng.to_device(np.zeros((n, 3)))
    g, _ = eng.imu_noise(FS, R, ref, ref, err, dict(err, vrw=err['arw']), SEED, layout=eng.LAYOUT_CHANNEL_MAJOR)
    import oracle_np as onp
    m = np.asarray(onp.allan_multipliers(n, FS), dtype=np.float64)
    for fn, expect in ((eng.allan, nz.allan_expect), (eng.oallan, nz.allan_expect),
                       (eng.ohadamard, nz.hadamard_expect)):
        v, _ = fn(FS, g, n, R * 3)
        v = v.cpu().numpy()
        want = expect(m, dt, **p)
        mean, se = v.mean(0), v.std(0) / math.sqrt(v.shape[0])
        assert np.all(np.abs(mean - want) <= 5.0 * se), (fn.__name__, (mean / want).round(4))
    if 'R' in p:
        v, _ = eng.ohadamard(FS, g, n, R * 3)
        want0 = nz.hadamard_expect(m, dt, **dict(p, R=0.0))
        np.testing.assert_allclose(v.cpu().numpy().mean(0) / want0, 1.0, atol=0.1)


# ---- free integration: K1 (with the terms) then K2 -------------------------------------------------------------
def _sim(rf, imu, force=False):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    g = load_golden('philox_90deg_mid_rf%d.npz' % rf)
    traj = {k: g[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    sim = Sim([100.0, 0.0, 0.0], traj, ref_frame=rf, imu=imu, algorithm=FreeIntegration(g['ini']),
              seed=int(g['seed']))
    sim._force_fed = force
    return sim, g


def _answers(sim, rf):
    out = {'end': sim.end_point_errors(), 'hist': sim.histories(imu=True, quat=True),
           'hist4': sim.histories(stride=4)}
    for dn in ('att_euler', 'pos', 'vel'):
        for start in (-1, 2.5):
            st = sim.get_error_stats(dn, start)
            out[(dn, start)] = {k: (np.stack([st[k][r] for r in sorted(st[k])]) if isinstance(st[k], dict)
                                    else st[k]) for k in ('max', 'avg', 'std')}
    if rf == 0:
        for opt in ('ned', 'ecef'):
            for start in (-1, 2.5):
                st = sim.get_error_stats('pos', start, extra_opt=opt)
                out[(opt, start)] = {k: (np.stack([st[k][r] for r in sorted(st[k])]) if isinstance(st[k], dict)
                                         else st[k]) for k in ('max', 'avg', 'std')}
    out['pos3'] = sim.get_data(['pos'])[0]['algo0_3']
    out['gyro5'] = sim.get_data(['gyro'])[0][5]
    return out


def _same(a, b, tol, what=''):
    if isinstance(a, dict):
        for k in a:
            _same(a[k], b[k], tol, '%s %s' % (what, k))
        return
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, what
    assert np.max(np.abs(a - b), initial=0.0) <= tol * max(1.0, np.max(np.abs(b), initial=0.0)), what


@pytest.mark.parametrize('rf', [1, 0])
def test_free_integration_route_without_terms_is_k12(eng, rf):
    from gnss_ins_sim_b200 import imu_model
    runs = 9
    answers = []
    for force in (False, True):
        sim, _ = _sim(rf, imu_model.IMU('mid-accuracy', gps=False), force)
        sim.run(runs)
        answers.append(_answers(sim, rf))
    k12, fed = answers
    end = k12['end'].copy()
    end[:, 0:3] = wrap_pi(fed['end'][:, 0:3] - end[:, 0:3]) + end[:, 0:3]
    _same(fed['end'], end, 1e-9, 'end')
    for k in k12:
        if k in ('end', 'hist', 'hist4'):
            continue
        # NED / ECEF metres are differences of ECEF coordinates of ~6.4e6 m: 1e-9 m is a few of their roundings
        _same(fed[k], k12[k], 1e-8 if k[0] in ('ned', 'ecef') else 1e-9, str(k))
    for h in ('hist', 'hist4'):
        for k in k12[h]:
            x, y = fed[h][k], k12[h][k]
            if k == 'att_euler':
                x = wrap_pi(x - y) + y
            _same(x, y, 1e-9, '%s %s' % (h, k))


@pytest.mark.parametrize('rf', [1, 0])
def test_free_integration_with_terms_is_k2_on_k1_ex(eng, rf):
    from gnss_ins_sim_b200 import imu_model
    acc = {'gyro_b': [0.0] * 3, 'gyro_b_stability': [3.5] * 3, 'gyro_arw': [0.25] * 3, 'gyro_b_corr': [100.0] * 3,
           'accel_b': [0.0] * 3, 'accel_b_stability': [5e-5] * 3, 'accel_vrw': [0.03] * 3,
           'accel_b_corr': [100.0] * 3, 'gyro_rrw': [50.0] * 3, 'gyro_q': [1e-3] * 3, 'gyro_rr': [20.0] * 3,
           'accel_rrw': [1.0] * 3, 'accel_q': [1e-3] * 3, 'accel_rr': [5.0] * 3}
    imu = imu_model.IMU(acc, gps=False)
    sim, g = _sim(rf, imu)
    R = 6
    sim.run(R)
    dev = eng.to_device
    gyro, accel = eng.imu_noise(100.0, R, dev(g['ref_gyro']), dev(g['ref_accel']), imu.gyro_err, imu.accel_err,
                                int(g['seed']))
    att, pos, vel = eng.free_integration(rf, 100.0, gyro, accel, dev(np.asarray(g['ini'])[None]))
    att, pos, vel = (t.cpu().numpy() for t in (att, pos, vel))
    end = np.concatenate([wrap_pi(att[:, -1] - g['ref_att'][-1]), pos[:, -1] - g['ref_pos'][-1],
                          vel[:, -1] - g['ref_vel'][-1]], axis=1)
    _same(sim.end_point_errors(), end, 1e-12, 'end')
    st = sim.get_error_stats('vel', -1)
    _same(st['std'], np.std(end[:, 6:9], 0), 1e-9, 'std')
    ps = sim.get_error_stats('pos', 2.5)
    e = pos[:, 250:] - g['ref_pos'][None, 250:]
    _same(np.stack([ps['avg']['algo0_%d' % r] for r in range(R)]), e.mean(1), 1e-12, 'proc avg')
    _same(sim.get_data(['vel'])[0]['algo0_4'], vel[4], 1e-12, 'history')
    _same(sim.get_data(['accel'])[0][2], accel[2].cpu().numpy(), 0.0, 'imu')
    h = sim.histories(imu=True)
    _same(h['pos'], pos, 1e-12, 'histories')
    _same(h['gyro'], gyro.cpu().numpy(), 0.0, 'histories imu')
    # the terms reach the sensor statistics (K9-ex)
    sg = sim.get_error_stats('gyro', -1)
    _same(sg['avg'], (gyro.cpu().numpy()[:, -1] - g['ref_gyro'][-1]).mean(0), 1e-12, 'gyro stats')
    # and Allan through Sim runs the materialised path on K1-ex's series
    from gnss_ins_sim_b200.allan_analysis import Allan
    from gnss_ins_sim_b200.sim import Sim
    traj = {k: g[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    s2 = Sim([100.0, 0.0, 0.0], traj, ref_frame=rf, imu=imu, algorithm=Allan(), seed=int(g['seed']))
    s2.run(R)
    gc = gyro.permute(0, 2, 1).contiguous()
    v, _ = eng.allan(100.0, gc, gc.shape[2], R * 3)
    ad = np.sqrt(v.cpu().numpy()).reshape(R, 3, -1).transpose(0, 2, 1)
    _same(np.stack([s2.get_data(['ad_gyro'])[0]['algo0_%d' % r] for r in range(R)]), ad, 1e-12, 'allan')


# ---- closure with the Allan noise identification (K13) ---------------------------------------------------------
def _law_sim(kind, R, seed):
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.allan_analysis import Allan
    from gnss_ins_sim_b200.sim import Sim
    n = nz.LAW_N
    imu = imu_model.IMU('mid-accuracy', gps=False)
    ge, ae = nz.law_errs(kind)
    imu.set_gyro_error(ge)        # the stored SI keys, as columns 0, 3 and 4 of noise_* would be passed back in
    imu.set_accel_error(ae)
    z = np.zeros((n, 3))
    traj = {'ref_pos': z, 'ref_vel': z, 'ref_att': z, 'ref_accel': np.tile([0.0, 0.0, -9.8], (n, 1)), 'ref_gyro': z}
    sim = Sim([nz.LAW_FS, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Allan(fit=True), seed=seed)
    sim.run(R)
    out = {w: np.stack([sim.get_data([w])[0]['algo0_%d' % r] for r in range(R)])
           for w in ('noise_gyro', 'noise_accel', 'ad_gyro', 'ad_accel')}
    return out, traj


def _coef(out):
    q, nn, b, k, r = out[:5]
    return np.array([3.0 * q * q, nn * nn, (b / af.B_SCALE) ** 2, k * k / 3.0, r * r / 2.0])


@pytest.mark.parametrize('kind', ['rrw', 'rr', 'q'])
def test_allan_fit_through_sim_is_the_oracle_fit_of_the_oracle_series(eng, kind):
    """Allan(fit=True) through Sim on K1-ex's series against allan_fit_np.fit of the oracle's series of the same
    runs: the same support and the coefficients to 1e-9.  Seed 3 keeps every channel's support clear of ties by
    more than 1e-9 of sum w (asserted), so that the support is decided."""
    import oracle_np as onp
    R, seed, n, fs = 2, 3, nz.LAW_N, nz.LAW_FS
    got, traj = _law_sim(kind, R, seed)
    ge, ae = nz.law_errs(kind)
    og, oa = nz.imu_noise(fs, traj['ref_gyro'], traj['ref_accel'], ge, ae, seed, np.arange(R))
    for which, series in (('gyro', og), ('accel', oa)):
        for r in range(R):
            for c in range(3):
                v = onp.allan_var(series[r, :, c], fs)[0]
                o, info = af.fit(v, n, fs, detail=True)
                d = np.array([ob - info['objective'] for m, ob in info['objectives'].items() if m != info['mask']])
                assert np.all((d > 1e-9 * info['W']) | (np.abs(d) < 1e-15 * info['W'])), (which, r, c)
                assert_close(got['ad_' + which][r, :, c], np.sqrt(v), 1e-9, 0.0, 'curve')
                C, Cg = info['C'], _coef(got['noise_' + which][r, c])
                assert np.array_equal(C > 0.0, Cg > 0.0), (which, r, c, C, Cg)
                assert np.all(np.abs(Cg - C) <= 1e-9 * C), (which, r, c, np.abs(Cg - C) / np.where(C > 0, C, 1.0))


@pytest.mark.parametrize('kind', ['rrw', 'rr', 'q'])
def test_identified_terms_inside_the_oracle_envelopes(eng, kind):
    """200 runs of the law cases (100 Hz, 360 000 samples) through Sim: the term Allan(fit=True) identifies on every
    gyro and accel channel inside the envelope noise952_np derives from its own generator, and the mean within 5
    standard errors of the oracle's."""
    got, _ = _law_sim(kind, 200, 11)
    c = nz.LAWS[kind]
    for which in ('noise_gyro', 'noise_accel'):
        ok, summary = nz.law_check(kind, got[which][:, :, c['col']] / c['truth'])
        assert ok, (which, summary, c)
