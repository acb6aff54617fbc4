"""Overlapping Hadamard variance (K4o's Hadamard form) without a GPU: the NumPy oracle against the definition,
the tau grid, closed forms (a linear drift cancels exactly), the IEEE non-finite cases, why the device prefix
has to be compensated, and the plugin's attributes and output names."""
import numpy as np
import pytest

import oallan_np as oa
import ohadamard_np as oh
import oracle_np as onp


@pytest.mark.parametrize('n, fs, seed', [(90, 1.0, 0), (1000, 10.0, 1), (1999, 100.0, 2), (2000, 3.0, 3)])
def test_oracle_matches_the_definition(n, fs, seed):
    x = np.random.default_rng(seed).standard_normal(n) * 0.1 + 2.0
    a, tau = oh.ohadamard_var(x, fs)
    b, tb = oh.ohadamard_var_brute(x, fs)
    m = onp.allan_multipliers(n, fs)
    assert len(a) == len(m) > 0 and np.array_equal(tau, tb)
    assert np.abs(a / b - 1.0).max() <= 1e-12


def test_tau_grid_is_the_reference_grid():
    for n, fs in [(90, 1.0), (8000, 100.0), (9000, 1.0), (123457, 200.0)]:
        x = np.random.default_rng(n).standard_normal(n)
        _, tau = oh.ohadamard_var(x, fs)
        _, t_ref = onp.allan_var(x, fs)
        assert tau.size > 0 and np.array_equal(tau, t_ref)
    assert oh.ohadamard_var(np.ones(800), 100.0)[0].size == 0     # too short: the reference's empty result
    assert oh.ohadamard_var_brute(np.ones(8), 1.0)[0].size == 0


def test_closed_forms():
    assert np.all(oh.ohadamard_var(np.full(3000, -7.25), 10.0)[0] == 0.0)
    n = 4500
    m = np.asarray(onp.allan_multipliers(n, 1.0), dtype=np.float64)
    for b in (3.0, -7.0):
        ramp = b * np.arange(n)
        # a linear drift cancels exactly in the second difference; the Allan variance keeps b^2 m^2 / 2
        assert np.all(oh.ohadamard_var(ramp, 1.0)[0] == 0.0)
        av, _ = oa.oallan_var(ramp, 1.0)
        assert np.abs(av / (b * b * m * m / 2.0) - 1.0).max() <= 1e-12
    # x_i = q i^2: the third difference of the cubic prefix is 2 q m^3, so hvar = (2/3) q^2 m^4
    q = 3.0
    hv, _ = oh.ohadamard_var(q * np.arange(n) ** 2, 1.0)
    assert np.abs(hv / (2.0 / 3.0 * q * q * m ** 4) - 1.0).max() <= 1e-12


def _nan_by_rule(x, fs):
    """The non-finite rule of K4o's Hadamard form, from +inf / -inf window counts: a term is NaN exactly when
    its contributions +S(k+2m), -2 S(k+m), +S(k) hold both infinities."""
    n = len(x)
    cp = np.concatenate([[0], np.cumsum(x == np.inf)])
    cn = np.concatenate([[0], np.cumsum(x == -np.inf)])
    out = []
    for m in onp.allan_multipliers(n, fs):
        k = np.arange(n - 3 * m + 1)
        p = [cp[k + (i + 1) * m] - cp[k + i * m] > 0 for i in range(3)]
        q = [cn[k + (i + 1) * m] - cn[k + i * m] > 0 for i in range(3)]
        pos = p[2] | q[1] | p[0]
        neg = q[2] | p[1] | q[0]
        out.append((pos & neg).any())
    return np.array(out)


def test_non_finite_samples_follow_ieee_arithmetic():
    rng = np.random.default_rng(5)
    n = 400
    m = np.asarray(onp.allan_multipliers(n, 1.0))
    x = rng.standard_normal(n)
    x[123] = np.nan
    assert np.isnan(oh.ohadamard_var_brute(x, 1.0)[0]).all() and np.isnan(oh.ohadamard_var(x, 1.0)[0]).all()
    x = rng.standard_normal(n)
    x[7] = np.inf
    assert (oh.ohadamard_var_brute(x, 1.0)[0] == np.inf).all()
    j = list(m).index(5)
    cases = [
        # a window holds both signs: NaN once m > d
        ([(200, np.inf), (201, -np.inf)], None),
        ([(200, np.inf), (204, -np.inf)], None),
        # S2 and S0 infinite with opposite signs, S1 finite: d = 2m puts them there at m = 5
        ([(100, np.inf), (110, -np.inf)], 'nan'),
        # S2 and S0 infinite with the same sign: +inf at m = 5 (no term puts them in adjacent windows)
        ([(100, np.inf), (110, np.inf)], 'inf'),
        # S1 infinite with the sign of S2 (or of S0): d = m
        ([(100, -np.inf), (105, -np.inf)], 'nan'),
        # opposite signs m apart: in adjacent windows they enter the term with one sign
        ([(100, np.inf), (105, -np.inf)], None),
        ([(0, -np.inf)], 'inf'), ([(399, np.inf)], 'inf'),
    ]
    for spots, at5 in cases:
        x = rng.standard_normal(n)
        for i, v in spots:
            x[i] = v
        b = oh.ohadamard_var_brute(x, 1.0)[0]
        assert np.array_equal(np.isnan(b), _nan_by_rule(x, 1.0)), spots
        assert (b[~np.isnan(b)] == np.inf).all(), spots
        if at5 is not None:
            assert (np.isnan(b[j]) if at5 == 'nan' else b[j] == np.inf), spots
        o = oh.ohadamard_var(x, 1.0)[0]
        assert np.array_equal(np.isnan(o), np.isnan(b)) and np.array_equal(o[~np.isnan(o)], b[~np.isnan(b)])
    # both signs in one window: NaN exactly where m exceeds their distance
    x = rng.standard_normal(n)
    x[200], x[204] = np.inf, -np.inf
    b = oh.ohadamard_var_brute(x, 1.0)[0]
    assert np.isnan(b[m > 4]).all()


def test_a_float64_prefix_misses_a_drifting_offset_series():
    """x_i = 1e4 + 1e-3 i + white noise of 1e-3, n = 1e6, m = 1, against the direct sum of the second
    differences: the long-double prefix holds it to 1e-10, a plain float64 prefix is far off.  The GPU tests
    hold the device to 1e-9 on this series, so they separate a compensated prefix from a naive one."""
    n = 10 ** 6
    x = 1e4 + 1e-3 * np.arange(n) + 1e-3 * np.random.default_rng(1).standard_normal(n)
    d = x[2:] - 2.0 * x[1:-1] + x[:-2]
    direct = np.sum(d * d) / (6.0 * (n - 2))
    ld = oh.ohadamard_var(x, 100.0)[0][0]
    f64 = oh.ohadamard_var_prefix64(x, 100.0)[0][0]
    assert abs(ld / direct - 1.0) < 1e-10
    assert abs(f64 / direct - 1.0) > 1e-8
    # the exact fixed-point form: the direct sum at m = 1; at long tau, where the drift cancels but the
    # prefix does not, it separates from the long-double form, which still holds every tau up to 10^4
    ex, tau = oh.ohadamard_var_fixed(x, 100.0)
    assert abs(ex[0] / direct - 1.0) < 1e-10
    m = np.rint(tau * 100.0)
    ld = oh.ohadamard_var(x, 100.0)[0]
    assert np.abs(ld / ex - 1.0)[m <= 10 ** 4].max() < 1e-9 and np.abs(ld / ex - 1.0).max() > 1e-9


def test_fixed_point_form_is_the_prefix_form_on_grid_series():
    rng = np.random.default_rng(8)
    for n, off, scale in ((2000, 3.0, 1e-3), (9000, -1e4, 0.5), (50000, 1e4, 1e-3)):
        x = off + scale * rng.standard_normal(n) + 1e-4 * np.arange(n) / n
        x = np.ldexp(np.rint(np.ldexp(x, 30)), -30)        # on a grid of 2^-30: x - x_0 exact
        ex, t1 = oh.ohadamard_var_fixed(x, 10.0)
        ld, t2 = oh.ohadamard_var(x, 10.0)
        assert np.array_equal(t1, t2) and np.abs(ex / ld - 1.0).max() < 1e-12
    with pytest.raises(ValueError):
        oh.ohadamard_var_fixed(np.array([1.0, 1e-300] * 50), 1.0)


def test_hadamard_plugin_attributes():
    from gnss_ins_sim_b200.allan_analysis import Allan, Hadamard
    from gnss_ins_sim_b200 import logged
    h = Hadamard()
    assert h.input == ['fs', 'accel', 'gyro'] and h.output == ['algo_time', 'hd_accel', 'hd_gyro'] and h.batch
    assert h.get_results() is None and h.reset() is None
    assert Allan(overlapping=True).output == ['algo_time', 'ad_accel', 'ad_gyro']    # unchanged
    for name, sensor in (('hd_gyro', 'gyro'), ('hd_accel', 'accel')):
        legend, units, out_units = logged.output_format(name, 0)
        assert legend == ['HD_%s_%s' % (sensor, c) for c in 'xyz']
        assert (units, out_units) == logged.output_format('ad_' + sensor, 0)[1:]
