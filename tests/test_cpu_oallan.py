"""Overlapping Allan variance (K4o) without a GPU: the NumPy oracle against the definition, closed
forms, the non-finite cases, why the device prefix has to be compensated, and the plugin's flag."""
import numpy as np
import pytest

import oallan_np as oa
import oracle_np as onp


@pytest.mark.parametrize('n, fs, seed', [(90, 1.0, 0), (1000, 10.0, 1), (1999, 100.0, 2), (2000, 3.0, 3)])
def test_oracle_matches_the_definition(n, fs, seed):
    x = np.random.default_rng(seed).standard_normal(n) * 0.1 + 2.0
    a, tau = oa.oallan_var(x, fs)
    b, tb = oa.oallan_var_brute(x, fs)
    m = onp.allan_multipliers(n, fs)
    assert len(a) == len(m) > 0 and np.array_equal(tau, tb)
    assert np.abs(a / b - 1.0).max() <= 1e-12


def test_tau_grid_is_the_reference_grid():
    for n, fs in [(100, 1.0), (800, 100.0), (9000, 1.0), (123457, 200.0), (14400000, 400.0)]:
        m = onp.allan_multipliers(n, fs)
        x = np.zeros(min(n, 200000))
        if len(x) == n:
            _, tau = oa.oallan_var(x, fs)
            assert np.array_equal(tau, np.asarray(m, dtype=np.float64) * (1.0 / fs))
    assert oa.oallan_var(np.ones(800), 100.0)[0].size == 0     # too short: the reference's empty result


def test_closed_forms():
    assert np.all(oa.oallan_var(np.full(3000, -7.25), 10.0)[0] == 0.0)
    n, a = 4500, 0.37
    av, tau = oa.oallan_var(a * np.arange(n), 1.0)
    m = np.asarray(onp.allan_multipliers(n, 1.0), dtype=np.float64)
    assert np.abs(av / ((a * m) ** 2 / 2.0) - 1.0).max() <= 1e-12
    # ... and the definition gives the same
    b, _ = oa.oallan_var_brute(a * np.arange(n), 1.0)
    assert np.abs(b / ((a * m) ** 2 / 2.0) - 1.0).max() <= 1e-12


def test_non_finite_samples_follow_ieee_arithmetic():
    rng = np.random.default_rng(5)
    n = 400
    m = np.asarray(onp.allan_multipliers(n, 1.0))
    x = rng.standard_normal(n)
    x[123] = np.nan
    assert np.isnan(oa.oallan_var_brute(x, 1.0)[0]).all() and np.isnan(oa.oallan_var(x, 1.0)[0]).all()
    x = rng.standard_normal(n)
    x[7] = np.inf
    assert (oa.oallan_var_brute(x, 1.0)[0] == np.inf).all()
    for d in (1, 4, 13):
        x = rng.standard_normal(n)
        x[200], x[200 + d] = np.inf, -np.inf
        b = oa.oallan_var_brute(x, 1.0)[0]
        assert np.isnan(b[m > d]).all() and (b[m <= d] == np.inf).all(), d
        o = oa.oallan_var(x, 1.0)[0]
        assert np.array_equal(np.isnan(o), np.isnan(b)) and np.array_equal(o[~np.isnan(o)], b[~np.isnan(b)])
    # two infinities of one sign d apart: NaN once a term can hold one in each window (2m > d)
    x = rng.standard_normal(n)
    x[50], x[50 + 30] = np.inf, np.inf
    b = oa.oallan_var_brute(x, 1.0)[0]
    assert np.isnan(b[2 * m > 30]).all() and (b[2 * m <= 30] == np.inf).all()


def test_a_float64_prefix_misses_a_drifting_series():
    """x_i = 1e4 + 1e-3 i + white noise of 1e-3, n = 1e6, m = 1, against the direct sum of the m = 1
    differences: the long-double prefix holds it to ~1e-11, a plain float64 prefix is off by ~3e-8.
    The GPU tests hold K4o to 1e-9 on this series, so they separate a compensated prefix from a naive one."""
    n = 10 ** 6
    x = 1e4 + 1e-3 * np.arange(n) + 1e-3 * np.random.default_rng(1).standard_normal(n)
    d = np.diff(x)
    direct = np.sum(d * d) / (2.0 * (n - 1))
    ld = oa.oallan_var(x, 100.0)[0][0]
    f64 = oa.oallan_var_prefix64(x, 100.0)[0][0]
    assert abs(ld / direct - 1.0) < 1e-10
    assert abs(f64 / direct - 1.0) > 1e-8


def test_allan_overlapping_argument():
    from gnss_ins_sim_b200.allan_analysis import Allan
    assert Allan().overlapping is False
    assert Allan(overlapping=True).overlapping is True
    assert Allan(np.bool_(True)).overlapping is True
    a = Allan(overlapping=True)
    assert a.input == ['fs', 'accel', 'gyro'] and a.output == ['algo_time', 'ad_accel', 'ad_gyro'] and a.batch
    for bad in (1, 'yes', None, 0.0):
        with pytest.raises(TypeError):
            Allan(overlapping=bad)
