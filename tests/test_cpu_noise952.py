"""IEEE Std 952 terms of the IMU model (quantisation, rate random walk, rate ramp) without a GPU: the IMU's units
and keys, the C struct, the oracle (oracle/noise952_np.py) and its exact Allan and Hadamard expectations, and
the plugins that cannot take the terms."""
import ctypes
import math
import os

import numpy as np
import pytest

import noise952_np as nz
import oracle_np as onp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D2R = math.pi / 180.0
BASE = {'gyro_b': [0.0] * 3, 'gyro_b_stability': [1.0] * 3, 'gyro_arw': [0.1] * 3, 'gyro_b_corr': [100.0] * 3,
        'accel_b': [0.0] * 3, 'accel_b_stability': [1e-4] * 3, 'accel_vrw': [0.05] * 3, 'accel_b_corr': [100.0] * 3}


def test_imu_terms_in_si_units():
    from gnss_ins_sim_b200.imu_model import IMU
    imu = IMU(dict(BASE, gyro_q=[2.0, 2.0, 2.0], gyro_rrw=[3.0, 3.0, 3.0], gyro_rr=[4.0, 4.0, 4.0],
                   accel_q=0.01, accel_rrw=[0.6, 0.6, 0.6], accel_rr=[36.0, 36.0, 36.0]))
    np.testing.assert_allclose(imu.gyro_err['q'], 2.0 * D2R, rtol=1e-15)
    np.testing.assert_allclose(imu.gyro_err['rrw'], 3.0 * D2R / 3600.0 / math.sqrt(3600.0), rtol=1e-15)
    np.testing.assert_allclose(imu.gyro_err['rr'], 4.0 * D2R / 3600.0 ** 2, rtol=1e-15)
    np.testing.assert_allclose(imu.accel_err['q'], [0.01] * 3, rtol=1e-15)
    np.testing.assert_allclose(imu.accel_err['rrw'], 0.6 / 60.0, rtol=1e-15)
    np.testing.assert_allclose(imu.accel_err['rr'], 36.0 / 3600.0, rtol=1e-15)
    # absent keys are not stored; the string grades gain no keys
    only = IMU(dict(BASE, gyro_rrw=[1.0] * 3))
    assert 'rrw' in only.gyro_err and 'q' not in only.gyro_err and not {'q', 'rrw', 'rr'} & set(only.accel_err)
    for grade in ('low-accuracy', 'mid-accuracy', 'high-accuracy'):
        g = IMU(grade)
        assert set(g.gyro_err) == {'b', 'b_drift', 'b_corr', 'arw'} and set(g.accel_err) == {'b', 'b_drift',
                                                                                              'b_corr', 'vrw'}
    assert set(IMU(dict(BASE)).gyro_err) == {'b', 'b_drift', 'b_corr', 'arw'}


def test_imu_term_keys_are_validated():
    from gnss_ins_sim_b200.imu_model import IMU
    for key, bad in (('gyro_q', -1.0), ('gyro_rrw', float('nan')), ('accel_q', float('inf')), ('accel_rrw', -0.1),
                     ('gyro_rr', float('inf'))):
        with pytest.raises(ValueError, match=key):
            IMU(dict(BASE, **{key: [bad] * 3}))
    IMU(dict(BASE, gyro_rr=[-1.0] * 3))          # a ramp may have either sign
    imu = IMU('mid-accuracy')
    imu.set_gyro_error({'q': np.full(3, 1e-6), 'rrw': np.full(3, 2e-6), 'rr': np.full(3, 3e-7)})
    imu.set_accel_error({'rrw': np.full(3, 1e-4)})
    assert imu.gyro_err['rrw'][0] == 2e-6 and imu.accel_err['rrw'][0] == 1e-4
    with pytest.raises(ValueError, match='unsupported key'):
        imu.set_gyro_error({'rrw_x': 1.0})


def test_noise_terms_struct_matches_header():
    from gnss_ins_sim_b200 import _lib
    assert ctypes.sizeof(_lib.NoiseTerms) == 72
    assert (_lib.NoiseTerms.q.offset, _lib.NoiseTerms.k.offset, _lib.NoiseTerms.r.offset) == (0, 24, 48)
    assert ctypes.sizeof(_lib.SensorErr) == 96
    with open(os.path.join(ROOT, 'include', 'b2ins.h')) as f:
        h = f.read()
    assert 'typedef struct b2ins_noise_terms {\n  double q[3];\n  double k[3];\n  double r[3];\n} b2ins_noise_terms;' in h
    # a dict without a non-zero term passes NULL: the entry points then launch the kernels without terms
    assert _lib.noise_terms({'b': 0}) is None and _lib.noise_terms({'q': np.zeros(3), 'rr': 0.0}) is None
    t = _lib.noise_terms({'rrw': np.array([1.0, 2.0, 3.0]), 'rr': 0.5})
    assert list(t.k) == [1.0, 2.0, 3.0] and list(t.r) == [0.5] * 3 and list(t.q) == [0.0] * 3


def _errs(**kw):
    g = {'b': np.array([1e-4, 0.0, -2e-4]), 'b_drift': np.full(3, 1e-5), 'b_corr': np.array([100.0, np.inf, 5.0]),
         'arw': np.full(3, 1e-4)}
    a = {'b': np.array([0.01, 0.0, -0.02]), 'b_drift': np.full(3, 1e-3), 'b_corr': np.array([np.inf, 50.0, 1.0]),
         'vrw': np.full(3, 1e-3)}
    return dict(g, **kw), dict(a, **kw)


def test_oracle_with_zero_terms_is_oracle_np():
    n = 300
    rng = np.random.default_rng(3)
    rg, ra = rng.standard_normal((n, 3)), rng.standard_normal((n, 3))
    ge, ae = _errs(q=np.zeros(3), rrw=np.zeros(3), rr=np.zeros(3))
    g0, a0 = onp.imu_noise(100.0, rg, ra, ge, ae, 9, [0, 5, 2 ** 33])
    g1, a1 = nz.imu_noise(100.0, rg, ra, ge, ae, 9, [0, 5, 2 ** 33])
    assert np.array_equal(g0, g1) and np.array_equal(a0, a1)


def test_oracle_terms_follow_their_definition():
    fs, n = 50.0, 40
    dt = 1.0 / fs
    err = {'q': np.array([1e-3, 2e-3, 0.0]), 'rrw': np.array([0.0, 1e-2, 3e-2]), 'rr': np.array([1e-3, 0.0, -2e-3])}
    walk, quant, ramp = nz.term_parts(fs, n, err, 1, 77, [4, 2 ** 32 + 1])
    for ri, run in enumerate([4, 2 ** 32 + 1]):
        for c in range(3):
            z0 = np.array([onp.normal_pair(t, nz.DRAW_RRW + 3 + c, run, 77)[0] for t in range(n)])
            w = np.zeros(n)
            for t in range(n - 1):
                w[t + 1] = w[t] + err['rrw'][c] * math.sqrt(dt) * z0[t]
            np.testing.assert_allclose(walk[ri, :, c], w, rtol=1e-13, atol=1e-18)
            u = np.array([nz.uniform01(t, nz.DRAW_QUANT + 3 + c, run, 77) for t in range(n + 1)])
            assert np.all((u >= 0.0) & (u < 1.0))
            e = err['q'][c] * math.sqrt(12.0) * (u - 0.5)
            assert np.array_equal(quant[ri, :, c], (e[1:] - e[:-1]) / dt)
            assert np.array_equal(ramp[ri, :, c], err['rr'][c] * (np.arange(n) * dt))
    assert walk[:, 0].max() == 0.0


@pytest.mark.parametrize('kind', ['allan', 'hadamard'])
def test_closed_forms_equal_the_sums_over_the_weights(kind):
    dt = 0.01
    f = nz.allan_expect if kind == 'allan' else nz.hadamard_expect
    for m in (1, 2, 3, 7, 10, 64, 500):
        for p in ({'N': 1e-3}, {'Q': 2e-5}, {'K': 3e-4}, {'R': 1e-5}, {'N': 1e-3, 'Q': 2e-5, 'K': 3e-4, 'R': 1e-5}):
            np.testing.assert_allclose(f(m, dt, **p), nz.expect_by_sums(m, dt, kind, **p), rtol=1e-12, atol=1e-40)
    # the ramp vanishes from the Hadamard variance, and the walk's continuous-time limits
    assert nz.hadamard_expect(10, dt, R=1.0) == 0.0
    np.testing.assert_allclose(nz.allan_expect(10 ** 6, dt, K=1.0) / (10 ** 6 * dt / 3.0), 1.0, rtol=1e-11)
    np.testing.assert_allclose(nz.hadamard_expect(10 ** 6, dt, K=1.0) / (10 ** 6 * dt / 6.0), 1.0, rtol=1e-11)


def _ensemble(series, m, kind):
    """Every overlapping Allan or Hadamard difference of window m of each series: [S, H]."""
    c = np.cumsum(np.concatenate([np.zeros((series.shape[0], 1)), series], axis=1), axis=1)
    s = lambda k: (c[:, k + m:c.shape[1] - (2 * m if kind == 'hadamard' else m) + k] - c[:, k:c.shape[1] - m - (2 * m if kind == 'hadamard' else m) + k]) / m  # noqa: E731,E501
    if kind == 'allan':
        return (s(m) - s(0)) ** 2 / 2.0
    return (s(2 * m) - 2.0 * s(m) + s(0)) ** 2 / 6.0


@pytest.mark.parametrize('kind', ['allan', 'hadamard'])
@pytest.mark.parametrize('term', ['Q', 'K', 'R', 'all'])
def test_closed_forms_against_a_brute_force_ensemble(kind, term):
    """Series of the model drawn with NumPy (same definitions, another generator): the mean of the first
    difference over the ensemble within 5 standard errors of the closed form, at several m."""
    fs, n, S = 100.0, 64, 20000
    dt = 1.0 / fs
    p = {'Q': 2e-4, 'K': 5e-2, 'R': 3e-2, 'N': 1e-3}
    if term != 'all':
        p = {term: p[term]}
    rng = np.random.default_rng(11)
    y = np.zeros((S, n))
    if 'N' in p:
        y += p['N'] / math.sqrt(dt) * rng.standard_normal((S, n))
    if 'Q' in p:
        e = p['Q'] * math.sqrt(12.0) * (rng.random((S, n + 1)) - 0.5)
        y += (e[:, 1:] - e[:, :-1]) / dt
    if 'K' in p:
        y[:, 1:] += np.cumsum(p['K'] * math.sqrt(dt) * rng.standard_normal((S, n - 1)), axis=1)
    if 'R' in p:
        y += p['R'] * np.arange(n) * dt
    f = nz.allan_expect if kind == 'allan' else nz.hadamard_expect
    for m in (1, 2, 5, 10):
        d = _ensemble(y, m, kind)[:, 0]
        want = f(m, dt, **p)
        if want == 0.0:
            assert np.max(np.abs(d)) < 1e-20
            continue
        # a ramp alone is deterministic: every difference is the expectation, up to rounding
        assert abs(d.mean() - want) <= 5.0 * d.std() / math.sqrt(S) + 1e-9 * want, (m, d.mean(), want)


@pytest.mark.parametrize('plugin', ['ins_loose', 'odo'])
def test_sim_refuses_plugins_whose_kernels_make_no_terms(plugin):
    from gnss_ins_sim_b200.imu_model import IMU
    from gnss_ins_sim_b200.sim import Sim
    n = 8
    traj = {k: np.zeros((n, 3)) for k in ('ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    traj['ref_odo'] = np.zeros(n)
    if plugin == 'ins_loose':
        from gnss_ins_sim_b200.ins_loose import InsLoose
        algo = InsLoose(np.zeros(9))
    else:
        from gnss_ins_sim_b200.free_integration_odo import FreeIntegration as FreeIntegrationOdo
        algo = FreeIntegrationOdo(np.zeros(9))
    imu = IMU(dict(BASE, gyro_rrw=[1.0] * 3), odo=True)
    sim = Sim(100.0, traj, imu=imu, algorithm=algo)
    with pytest.raises(ValueError, match='rate random walk') as e:
        sim.run(1)
    assert 'gyro rrw' in str(e.value)
    assert 'gyro' not in sim.data and 'accel' not in sim.data      # refused before anything was reset


def test_law_series_are_the_generators():
    """law_gyro builds the law cases from the gyro draws alone: the gyro series imu_noise makes, bit for bit."""
    fs, n = 100.0, 500
    for kind in nz.LAWS:
        ge, ae = nz.law_errs(kind)
        g, _ = nz.imu_noise(fs, np.zeros((n, 3)), np.zeros((n, 3)), ge, ae, 3, [0, 7])
        assert np.array_equal(nz.law_gyro(kind, 3, [0, 7], fs, n), g), kind


@pytest.mark.parametrize('kind', ['rrw', 'rr', 'q'])
def test_law_envelopes_regenerate(kind):
    """The stored law statistics against 16 fresh runs of the generator (runs 1000.., another stretch of the
    stream): every ratio inside the envelope, the mean within 5 standard errors."""
    ok, summary = nz.law_check(kind, nz.law_ratios(kind, 1, np.arange(1000, 1016)))
    assert ok, (summary, nz.LAWS[kind])
