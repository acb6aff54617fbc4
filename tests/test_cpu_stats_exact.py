"""The exact statistics reference (oracle/stats_exact.py) against NumPy's np.max(np.abs(x)), np.average and
np.std, and the host merge of shard statistics (dist.merge_stats) with non-finite shards.  No GPU."""
from fractions import Fraction

import numpy as np
import pytest

import stats_exact as sx
from gnss_ins_sim_b200 import dist


def _numpy(x, axis=0):
    with np.errstate(invalid='ignore'):
        return np.stack([np.max(np.abs(x), axis), np.average(x, axis), np.std(x, axis)])


def _ulps(a, b):
    return np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


def test_fraction_arithmetic_restated():
    """The integer form equals the Fraction definition, rounded once."""
    rng = np.random.default_rng(1)
    v = np.concatenate([rng.standard_normal(37) * 1e-3 + 5.0, [1e-300, 3e5]])
    fr = [Fraction(float(a)) for a in v]
    mean = sum(fr) / len(fr)
    var = sum((a - mean) ** 2 for a in fr) / len(fr)
    got = sx.stats(v)
    assert got[1] == float(mean) and got[0] == np.max(np.abs(v))
    # the correctly rounded square root of var: s^2 <= var < next^2 around it
    s = Fraction(float(got[2]))
    lo, hi = Fraction(float(np.nextafter(got[2], 0))), Fraction(float(np.nextafter(got[2], np.inf)))
    assert ((lo + s) / 2) ** 2 <= var <= ((s + hi) / 2) ** 2


@pytest.mark.parametrize('n', [1, 2, 3, 100, 4097])
def test_agrees_with_numpy_to_one_ulp(n):
    """Benign columns (unit-variance data with an offset of a few standard deviations): np.average and np.std
    of a contiguous column (pairwise summation) are within one ulp of the exact values."""
    rng = np.random.default_rng(n)
    x = rng.standard_normal((5, n)) * np.array([[1e-3], [1.0], [7.0], [1e4], [0.5]]) + np.array(
        [[2e-3], [-3.0], [10.0], [0.0], [1.0]])
    got = sx.stats(x, axis=1)
    ref = _numpy(x, 1)
    assert np.array_equal(got[0], ref[0])
    assert _ulps(got[1], ref[1]).max() <= 1.0
    sd = ref[2] > 0
    assert np.array_equal(got[2][~sd], ref[2][~sd])
    assert _ulps(got[2][sd], ref[2][sd]).max(initial=0.0) <= 1.0


def test_small_cases():
    assert np.array_equal(sx.stats(np.array([[2.5]])), [[2.5], [2.5], [0.0]])
    assert np.array_equal(sx.stats(np.full((9, 1), -0.1)), [[0.1], [-0.1], [0.0]])
    assert np.array_equal(sx.stats(np.array([[1.0], [3.0]])), [[3.0], [2.0], [1.0]])
    assert np.isnan(sx.stats(np.zeros((0, 2)))).all()


def test_offset_dominated_beats_numpy():
    """D + sigma z with D / sigma = 1e9: NumPy's float64 std is ~1e-7 off there; the exact value is not."""
    rng = np.random.default_rng(3)
    z = rng.standard_normal(1000)
    x = 1e6 + 1e-3 * z
    fr = [Fraction(float(a)) for a in x]
    mean = sum(fr) / len(fr)
    var = sum((a - mean) ** 2 for a in fr) / len(fr)
    st = sx.stats(x)
    assert st[1] == float(mean)
    assert abs(st[2] ** 2 - float(var)) <= 4 * np.spacing(float(var))


@pytest.mark.parametrize('case', ['nan', '+inf', '-inf', 'both', 'nan_and_inf', 'all_nan'])
def test_non_finite_like_numpy(case):
    rng = np.random.default_rng(7)
    x = rng.standard_normal((50, 4))
    put = {'nan': [(3, 1, np.nan)], '+inf': [(49, 2, np.inf)], '-inf': [(0, 0, -np.inf)],
           'both': [(5, 3, np.inf), (6, 3, -np.inf)], 'nan_and_inf': [(5, 3, np.inf), (9, 3, np.nan)],
           'all_nan': [(i, 1, np.nan) for i in range(50)]}[case]
    for i, j, v in put:
        x[i, j] = v
    got, ref = sx.stats(x), _numpy(x)
    assert np.array_equal(np.isnan(got), np.isnan(ref)), (got, ref)
    assert np.array_equal(got[np.isinf(ref)], ref[np.isinf(ref)])
    clean = [j for j in range(4) if j not in {p[1] for p in put}]
    assert np.array_equal(got[:, clean], sx.stats(x[:, clean]))
    assert np.isfinite(got[:, clean]).all()


def test_assert_stats_catches_a_wrong_std_and_a_lost_nan():
    rng = np.random.default_rng(2)
    x = rng.standard_normal((200, 3)) + 5.0
    ref = sx.stats(x)
    sx.assert_stats(ref, ref, 64 * sx.EPS * np.abs(x).max(0), 1e-13)
    bad = ref.copy()
    bad[2, 1] *= 1 + 1e-10
    with pytest.raises(AssertionError):
        sx.assert_stats(bad, ref, 64 * sx.EPS * np.abs(x).max(0), 1e-13)
    x[7, 2] = np.nan
    with pytest.raises(AssertionError, match='NaN'):
        sx.assert_stats(ref, sx.stats(x), 64 * sx.EPS * np.abs(x).max(0), 1e-13)


def _blocks(x, cuts):
    out = []
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        s = _numpy(x[lo:hi]) if hi > lo else np.zeros((3, x.shape[1]))
        out.append((hi - lo, s[0], s[1], s[2]))
    return out


@pytest.mark.parametrize('case', ['nan', '+inf', '-inf', 'both_signs_apart', 'empty_shard'])
def test_merge_stats_non_finite_shards(case):
    """dist.merge_stats of per-shard NumPy statistics == NumPy's statistics of the union: NaN exactly where it
    is NaN, infinities equal, finite columns within 1e-13 of the exact values (Chan's update is as good as two
    passes)."""
    rng = np.random.default_rng(11)
    x = rng.standard_normal((90, 5)) * [1.0, 1e-3, 10.0, 1.0, 2.0] + [0.0, 1.0, -3.0, 1e3, 0.5]
    cuts = [0, 30, 61, 90]
    if case == 'nan':
        x[40, 2] = np.nan
    elif case == '+inf':
        x[65, 0] = np.inf
    elif case == '-inf':
        x[3, 4] = -np.inf
    elif case == 'both_signs_apart':
        x[3, 1], x[80, 1] = np.inf, -np.inf
    else:
        cuts = [0, 30, 30, 90]
    merged, n = dist.merge_stats(_blocks(x, cuts))
    assert n == 90
    ref = sx.stats(x)
    sx.assert_stats(merged, ref, 64 * sx.EPS * np.where(np.isfinite(x), np.abs(x), 0).max(0), 1e-13, 'merge ' + case,
                    'first')


def test_merge_stats_one_shard_all_nan():
    x = np.random.default_rng(5).standard_normal((20, 2))
    x[10:, 1] = np.nan
    merged, _ = dist.merge_stats(_blocks(x, [0, 10, 20]))
    assert np.isnan(merged[:, 1]).all() and np.isfinite(merged[:, 0]).all()
