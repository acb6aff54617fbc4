"""The exact IEEE Std 952 terms and run-to-run errors (oracle/terms_exact.py), without a GPU.

The fma emulation is held to hand-checked cases, one of which a separate product and sum round differently; the
closed forms of quantisation and ramp equal noise952_np bit for bit (it rounds the same three and two operations);
the walk is a Fraction cumulative sum on short series, and its Psi bounds NumPy's rounded cumsum (noise952_np's
walk: each step rounds K sqrt(dt) z and the sum, u |k z_s| + u |w[s+1]|, within u Psi_t to first order)."""
import math
from fractions import Fraction

import numpy as np
import pytest

import noise952_np as nz
import oracle_np as onp
import run_err_np as rx
import terms_exact as tx

U = 2.0 ** -53
FS = 100.0
SEED = 41
RUNS = np.array([3, 2 ** 32 - 1, 2 ** 32], dtype=np.uint64)


def test_fma_exact_cases():
    x = 1.0 + 2.0 ** -52
    assert tx.fma(x, 1.0 - 2.0 ** -52, -1.0) == -(2.0 ** -104)          # fused
    assert x * (1.0 - 2.0 ** -52) - 1.0 == 0.0                          # a product then a sum: another value
    assert tx.fma(0.1, 10.0, -1.0) == 2.0 ** -54
    assert 0.1 * 10.0 - 1.0 == 0.0
    assert tx.fma(3.0, 5.0, 7.0) == 22.0
    assert tx.fma(2.0 ** 1000, 2.0 ** 20, -(2.0 ** 1019)) == 2.0 ** 1019
    assert tx.fma(2.0 ** -1074, 0.5, 0.0) == 0.0                         # ties to even at the bottom
    assert tx.fma(2.0 ** -1074, 0.75, 0.0) == 2.0 ** -1074
    assert tx.fma(2.0 ** 1000, 2.0 ** 30, 0.0) == math.inf
    # exact zeros take IEEE's sign; non-finite operands propagate
    assert math.copysign(1.0, tx.fma(1.0, -1.0, 1.0)) == 1.0
    assert math.copysign(1.0, tx.fma(-0.0, 1.0, -0.0)) == -1.0
    assert math.isnan(tx.fma(0.0, math.inf, 1.0)) and math.isnan(tx.fma(0.0, 1.0, math.nan))
    assert math.isnan(tx.fma(0.0, math.nan, 1.0))                        # a zero entry of S times a NaN reference
    assert tx.fma(2.0, math.inf, 1.0) == math.inf
    # against Fraction on random operands, where the products are far from representable
    rng = np.random.default_rng(3)
    a, b, c = rng.standard_normal((3, 2000)) * np.array([[1.0], [1e-3], [1e-2]])
    got = tx.fma_np(a, b, c)
    want = np.array([float(Fraction(x) * Fraction(y) + Fraction(z)) for x, y, z in zip(a, b, c)])
    assert np.array_equal(got, want)
    assert np.count_nonzero(got != a * b + c) > 100                     # the fused results differ from NumPy's


def _err():
    return {'q': np.array([2e-5, 0.0, 3e-5]), 'rrw': np.array([3e-5, 1e-5, 0.0]), 'rr': np.array([1e-6, -2e-6, 0.0])}


def test_coefficients_are_digest_terms():
    q, k, r, dt = tx.coefficients(FS, _err())
    assert dt == 0.01
    assert np.array_equal(q, _err()['q'] * math.sqrt(12.0)) and np.array_equal(k, _err()['rrw'] * 0.1)
    assert np.array_equal(r, _err()['rr'])


@pytest.mark.parametrize('n', [1, 2, 7, 897])
def test_quantisation_and_ramp_are_noise952s(n):
    err = _err()
    q, k, r, dt = tx.coefficients(FS, err)
    for sensor in (0, 1):
        _, quant, ramp = nz.term_parts(FS, n, err, sensor, SEED, RUNS)
        u = tx.quant_uniforms(n, sensor, SEED, RUNS)
        assert np.all((u >= 0.0) & (u < 1.0)) and np.all(u * 2.0 ** 52 == np.floor(u * 2.0 ** 52))
        assert np.array_equal(tx.quant_rate(q, u, dt), quant)
        assert np.array_equal(np.broadcast_to(tx.ramp(r, n, dt), ramp.shape), ramp)
        assert np.all(tx.quant_rate(q, u, dt)[..., 1] == 0.0)          # q = 0: no quantisation


def _fraction_walk(k, z):
    K, W, out = Fraction(float(k)), Fraction(0), [0.0]
    for s in range(len(z) - 1):
        W += K * Fraction(float(z[s]))
        out.append(float(W))
    return np.array(out)


def test_walk_equals_fractions():
    rng = np.random.default_rng(5)
    z = rng.standard_normal((2, 300, 3))
    z[0, 7, 1] = 0.0
    z[1, 11, 2] = 2.0 ** -1070
    k = np.array([3e-6, 1.0, 0.0])
    d, psi = tx.walk(k, z)
    for r in range(2):
        for c in range(3):
            assert np.array_equal(d[r, :, c], _fraction_walk(k[c], z[r, :, c])), (r, c)
    assert np.all(d[:, :, 2] == 0.0) and np.all(psi[:, :, 2] == 0.0)
    assert np.all(psi >= np.abs(d)) and np.all(psi[:, 0] == 0.0)


def test_psi_bounds_numpys_cumsum():
    """noise952_np's walk on its own normals: within gamma_2 Psi of the exact walk, and outside u Psi / 4 at
    some sample (the bound is not slack by orders of magnitude)."""
    n, err = 20000, _err()
    _, k, _, _ = tx.coefficients(FS, err)
    for sensor in (0, 1):
        walk, _, _ = nz.term_parts(FS, n, err, sensor, SEED, RUNS)
        t = np.arange(n, dtype=np.uint64)[None, :, None]
        ax = np.arange(3, dtype=np.uint64)[None, None, :]
        z0, _ = onp.normal_pair(t, nz.DRAW_RRW + 3 * sensor + ax, RUNS[:, None, None], SEED)
        d, psi = tx.walk(k, z0)
        err_ = np.abs(walk - d)
        assert np.all(err_ <= tx.gamma(2) * psi)
        assert np.max(err_ / np.where(psi > 0, psi, np.inf)) > U / 4


def test_run_error_sample_is_the_fma_chain():
    """run_err_sample is ref + the kernel's fma chain; within gamma_4 of the exact b_run + S ref (and of
    run_err_np's delta, which rounds the products too).  Non-finite references as NumPy's ref + b + S @ ref has
    them: a NaN in one column makes all three channels of the sensor NaN (S[c][j] NaN is NaN even where S[c][j]
    is 0); an infinity makes all three non-finite, +-inf, or NaN where S[c][j] = 0 (0 inf) or on its own column
    when S[c][c] inf has the other sign."""
    rng = np.random.default_rng(9)
    ref = rng.standard_normal((40, 3)) * [0.1, 0.2, 9.8]
    err = {'b_std': np.array([1e-2, 3e-2, 0.0]), 'sf': np.array([3e-3, 0.0, 2e-3]), 'ma': 2e-3 * (1 - np.eye(3))}
    tab = rx.table(err, 0, SEED, RUNS)
    got = tx.run_err_sample(ref, tab)
    ex, env = tx.run_err_exact(ref, tab)
    assert np.all(np.abs(got - (ref[None] + ex)) <= tx.gamma(5) * (env + np.abs(ref)[None]))
    assert np.all(np.abs(ex - rx.delta(ref, tab)) <= tx.gamma(4) * env)
    for c in range(3):
        for r in range(len(RUNS)):
            for t in (0, 17):
                d = tab[r, c, 3]
                for j in range(3):
                    d = tx.fma(tab[r, c, j], ref[t, j], d)
                assert got[r, t, c] == ref[t, c] + d
    bad = ref.copy()
    bad[5, 1] = np.nan
    bad[6, 2] = np.inf
    g = tx.run_err_sample(bad, tab)
    assert np.isnan(g[:, 5]).all() and not np.isfinite(g[:, 6]).any()
    assert np.array_equal(g[:, :5], got[:, :5]) and np.array_equal(g[:, 7:], got[:, 7:])
    with np.errstate(invalid='ignore'):
        npy = bad[None] + rx.delta(bad, tab)
    assert np.array_equal(np.isnan(g), np.isnan(npy)) and np.array_equal(g[np.isinf(g)], npy[np.isinf(g)])
    # a zero entry of S meets the infinity: NaN there, as in NumPy
    tab0 = tab.copy()
    tab0[:, 0, 2] = 0.0
    g0 = tx.run_err_sample(bad, tab0)
    assert np.isnan(g0[:, 6, 0]).all() and np.isnan(g0[:, 5]).all()


def test_assemble_of_single_components():
    """With one component set the exact sum is that component, and the bound holds the rest of the sample at
    zero; with all of them the sum is the Fraction sum."""
    R, n = 2, 30
    rng = np.random.default_rng(2)
    z = rng.standard_normal((6, R, n, 3))
    zero = np.zeros((R, n, 3))
    ref = rng.standard_normal((n, 3))
    sens0 = {'b': np.zeros(3), 'w': np.zeros(3), 'wd': np.zeros(3)}
    tab0 = np.zeros((R, 3, 4))
    ex, bound = tx.assemble(np.zeros((n, 3)), sens0, z[0], z[1], zero, zero, zero, zero, zero, np.zeros((n, 3)), tab0,
                            916, 20)
    assert np.all(ex == 0.0) and np.all(bound == 0.0)
    ex, _ = tx.assemble(ref, sens0, z[0], z[1], zero, zero, zero, zero, z[2], np.zeros((n, 3)), tab0, 916, 20)
    assert np.array_equal(ex, ref[None] + z[2])
    sens = {'b': np.array([1e-3, 0.0, 2.0]), 'w': np.array([0.1, 0.2, 0.3]), 'wd': np.array([0.0, 1e-5, 0.0])}
    tab = rng.standard_normal((R, 3, 4)) * 1e-3
    ex, bound = tx.assemble(ref, sens, z[0], z[1], z[2], np.abs(z[2]), z[3], np.abs(z[3]), z[4], z[5, 0], tab, 916, 20)
    r, t, c = 1, 17, 2
    want = (Fraction(ref[t, c]) + Fraction(sens['b'][c]) + Fraction(sens['w'][c]) * Fraction(z[0, r, t, c]) +
            Fraction(sens['wd'][c]) * Fraction(z[1, r, t, c]) + Fraction(z[2, r, t, c]) + Fraction(z[3, r, t, c]) +
            Fraction(z[4, r, t, c]) + Fraction(z[5, 0, t, c]) + Fraction(tab[r, c, 3]) +
            sum(Fraction(tab[r, c, j]) * Fraction(ref[t, j]) for j in range(3)))
    assert ex[r, t, c] == float(want)
    assert np.all(bound > 0.0)
