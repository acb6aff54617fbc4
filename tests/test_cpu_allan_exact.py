"""The exact allan_var (oracle/allan_exact.py), the reference K4 is held to: against the definition in
Fractions, the float64 oracle, the reference's own results (allan.npz, allan_config4_full_length.npz) and
NumPy's NaN / inf class on a bank of non-finite cases.  No GPU."""
from fractions import Fraction

import numpy as np
import pytest

import allan_exact as ae
import oracle_np as onp
from conftest import assert_close, load_golden


def _fraction_allan(x, fs):
    """The definition in Fractions, one rounding at the end (finite x)."""
    n = len(x)
    out = []
    for m in onp.allan_multipliers(n, fs):
        nb = n // m
        means = [sum(Fraction(v) for v in x[b * m:(b + 1) * m]) / m for b in range(nb)]
        s = sum((means[b + 1] - means[b]) ** 2 for b in range(nb - 1))
        out.append(float(Fraction(1, 2 * (nb - 1)) * s))
    return np.array(out)


@pytest.mark.parametrize('case', ['noise', 'offset', 'tiny', 'mixed', 'constant'])
def test_exact_against_fractions(case):
    rng = np.random.default_rng(len(case))
    n = 1234
    x = {'noise': rng.standard_normal(n),
         'offset': 1e7 + rng.standard_normal(n),
         'tiny': 1e-300 * rng.standard_normal(n),
         'mixed': rng.standard_normal(n) * np.exp2(rng.integers(-60, 60, n)),
         'constant': np.full(n, 0.1)}[case]
    got, tau = ae.allan_var(x, 1.0)
    assert len(got) > 0 and np.array_equal(got, _fraction_allan(x, 1.0))
    assert np.array_equal(tau, np.asarray(onp.allan_multipliers(n, 1.0), dtype=np.float64) * 1.0)


@pytest.mark.parametrize('n,fs', [(9000, 1.0), (9009, 1.0), (50419, 100.0 / 3.0), (123457, 3.7), (1008001, 10.0)])
def test_exact_against_the_float64_oracle(n, fs):
    """The blocks of the exact form (1 008 000 samples) join without a seam."""
    x = np.random.default_rng(n).standard_normal(n) * 0.3 + 2.0
    ex, tau = ae.allan_var(x, fs)
    o, ot = onp.allan_var(x, fs)
    assert np.array_equal(tau, ot)
    assert_close(o, ex, 1e-12, 0.0, 'oracle_np against the exact form')


def test_tau_is_m_times_ts_bit_for_bit():
    """allan.py:58 forms tau = m * ts with ts = 1 / fs; m / fs differs in the last bit for some fs."""
    fs = 3.7
    mult = onp.allan_multipliers(90000, fs)
    _, tau = onp.allan_var(np.zeros(90000), fs)
    want = np.array([m * (1.0 / fs) for m in mult])
    assert np.array_equal(tau, want)
    assert not np.array_equal(want, np.array([m / fs for m in mult]))


def test_goldens():
    g = load_golden('allan.npz')
    for key, fs, a, t in (('x', 'fs', 'avar', 'tau'), ('x2', 'fs2', 'avar2', 'tau2')):
        ex, tau = ae.allan_var(g[key], float(g[fs]))
        assert np.array_equal(tau, g[t]), key
        assert_close(ex, g[a], 1e-12, 0.0, key)
    ex, tau = ae.allan_var(g['x3'], 100.0)
    assert len(ex) == 0 and len(tau) == 0


def test_config4_full_length_golden():
    """14.4 M samples at 400 Hz: the exact form against allan.allan_var of the unmodified reference."""
    import oracle_c
    from gnss_ins_sim_b200 import imu_model
    g = load_golden('allan_config4_full_length.npz')
    n, fs = int(g['n']), float(g['fs'])
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    og, oa = oracle_c.imu_noise(fs, np.zeros((n, 3)), np.tile(np.array([4.9, 0.0, -8.487]), (n, 1)),
                                imu.gyro_err, imu.accel_err, int(g['seed']), [int(g['run'])])
    ex, tau = ae.allan_var(np.ascontiguousarray(og[0, :, 2]), fs)
    assert_close(tau, g['tau'], 1e-15, 0.0, 'tau')
    assert_close(ex, g['avar_gyro_z'], 1e-10, 0.0, 'avar gyro z')
    ex, _ = ae.allan_var(np.ascontiguousarray(oa[0, :, 0]), fs)
    # (the reference's own float64 sums lose ~1e-8 of the accel x variance under its 4.9 m/s^2 offset)
    assert_close(ex, g['avar_accel_x'], 1e-7, 0.0, 'avar accel x')


def _bank(n):
    rng = np.random.default_rng(n)
    base = rng.standard_normal(n)
    cases = []
    top = onp.allan_multipliers(n, 1.0)[-1]
    for spots in ([(0, np.nan)], [(0, np.inf)], [(0, -np.inf)], [(0, np.inf), (1, -np.inf)],
                  [(n - 1, np.inf)], [(n - 1, np.nan)], [((n // top) * top, np.inf)],
                  [(100, np.inf), (101, np.inf)], [(100, np.inf), (102, np.inf)],
                  [(100, -np.inf), (103, -np.inf)], [(100, np.inf), (107, -np.inf)],
                  [(3, np.nan), (999, np.inf)], [(500, np.inf), (1500, -np.inf), (2500, np.nan)]):
        x = base.copy()
        for i, v in spots:
            x[i] = v
        cases.append(x)
    return cases


@pytest.mark.parametrize('n', [4001, 20011])
def test_non_finite_class_is_numpys(n):
    """NaN and +inf exactly where NumPy's evaluation of the reference's expression gives them; finite taus
    are those of the series with the changed samples left out."""
    for x in _bank(n):
        ex, _ = ae.allan_var(x, 1.0)
        with np.errstate(invalid='ignore', over='ignore'):
            o, _ = onp.allan_var(x, 1.0)
        assert np.array_equal(np.isnan(ex), np.isnan(o)), (x[np.isfinite(x) == 0], ex, o)
        assert np.array_equal(np.isinf(ex), np.isinf(o)) and not (ex == -np.inf).any()
        f = np.isfinite(ex)
        assert_close(ex[f], o[f], 1e-12, 0.0, 'finite taus beside non-finite samples')
    x = _bank(n)[6]                 # past nb * m of the longest tau: that tau stays finite
    assert np.isfinite(ae.allan_var(x, 1.0)[0][-1])
