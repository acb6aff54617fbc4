"""The Allan noise-identification oracle (oracle/allan_fit_np.py) on the CPU: against scipy's NNLS and an exact
rational solve, model curves of every support, the edge rules, the law envelopes the GPU tests reuse, the
Allan(fit=...) constructor and the argument checks of the K13 entry points (b2ins_allan_fit_f64 and its host twin)."""
import ctypes
from fractions import Fraction

import numpy as np
import pytest
from scipy.optimize import nnls

import allan_fit_np as af
import oracle_np

FS, N = 100.0, 360000
# model coefficients of a typical curve on the grid of (N, FS): each term matters somewhere on it
BASE_C = np.array([1e-8, 1e-6, 1e-8, 1e-10, 1e-13])


def _real_curves(seed, count):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(count):
        x = 1e-3 * np.sqrt(FS) * rng.standard_normal(N)
        x += np.cumsum(3e-5 * rng.uniform(0.3, 3.0) / np.sqrt(FS) * rng.standard_normal(N))
        x += rng.uniform(0.0, 2e-6) * np.arange(N) / FS
        out.append(oracle_np.allan_var(x, FS)[0])
    return out


def _random_curves(seed, count):
    rng = np.random.default_rng(seed)
    ntau = len(af.grid(N, FS)[0])
    return [af.model_curve(BASE_C * 10.0 ** rng.uniform(-1, 1, 5), N, FS) * np.exp(0.3 * rng.standard_normal(ntau))
            for _ in range(count)]


@pytest.mark.parametrize('kind', ['real', 'random'])
def test_oracle_is_the_nnls_optimum(kind):
    """scipy.optimize.nnls on the same scaled system: the same fitted model per bin and the same objective to
    1e-12 relative."""
    curves = _real_curves(1, 8) if kind == 'real' else _random_curves(2, 40)
    tau, w = af.grid(N, FS)
    for v in curves:
        out, info = af.fit(v, N, FS, detail=True)
        D, b, s, _ = af.system(v, tau, w)
        y, rnorm = nnls(D, b)
        ours = info['C'] * s
        assert np.all(np.abs(D @ ours - D @ y) <= 1e-12 * np.abs(D @ y)), (info['mask'], y, ours)
        assert abs(info['objective'] - rnorm ** 2) <= 1e-12 * info['W']
        assert np.all(info['C'] >= 0.0) and np.all(np.isfinite(out))


@pytest.mark.parametrize('seed', range(6))
def test_oracle_against_an_exact_rational_solve(seed):
    """The chosen support's coefficients against the exact least-squares solution (normal equations in Fraction)
    of the same float system, on a small grid (n = 900 at 10 Hz: 18 bins)."""
    n, fs = 900, 10.0
    rng = np.random.default_rng(seed)
    tau, w = af.grid(n, fs)
    x = rng.standard_normal(n) + np.cumsum(0.05 * rng.standard_normal(n)) + 0.002 * np.arange(n)
    v = oracle_np.allan_var(x, fs)[0]
    _, info = af.fit(v, n, fs, detail=True)
    D, b, s, _ = af.system(v, tau, w)
    cols = [i for i in range(5) if info['mask'] >> i & 1]
    assert cols
    A = [[Fraction(float(D[k, c])) for c in cols] for k in range(D.shape[0])]
    B = [Fraction(float(bk)) for bk in b]
    m = len(cols)
    M = [[sum(A[k][i] * A[k][j] for k in range(len(A))) for j in range(m)] + [sum(A[k][i] * B[k] for k in range(len(A)))]
         for i in range(m)]
    for i in range(m):                  # Gauss-Jordan, exact
        piv = next(r for r in range(i, m) if M[r][i] != 0)
        M[i], M[piv] = M[piv], M[i]
        for r in range(m):
            if r != i and M[r][i] != 0:
                f = M[r][i] / M[i][i]
                M[r] = [a - f * c for a, c in zip(M[r], M[i])]
    y = [M[i][m] / M[i][i] for i in range(m)]
    for i, c in enumerate(cols):
        exact = float(y[i]) / s[c]
        assert abs(info['C'][c] - exact) <= 1e-12 * exact, (c, info['C'][c], exact)


@pytest.mark.parametrize('mask', af.SUPPORTS)
def test_model_curves_of_every_support(mask):
    """sigma^2 built from known C on a support: the oracle picks that support, recovers C to 1e-12 relative and puts
    exact zeros off it."""
    rng = np.random.default_rng(mask)
    C = np.array([BASE_C[i] * 10.0 ** rng.uniform(-0.3, 0.3) if mask >> i & 1 else 0.0 for i in range(5)])
    out, info = af.fit(af.model_curve(C, N, FS), N, FS, detail=True)
    assert info['mask'] == mask
    on = C > 0.0
    assert np.all(np.abs(info['C'][on] - C[on]) <= 1e-12 * C[on]), (info['C'], C)
    assert np.all(info['C'][~on] == 0.0)
    want = af.outputs(C, af.model_curve(C, N, FS).min())
    assert np.all(np.abs(out - want) <= 1e-12 * want)
    assert np.all(out[:5][~on] == 0.0)


def test_edge_rules():
    ntau = len(af.grid(N, FS)[0])
    v = _random_curves(5, 1)[0]
    for bad in (np.nan, np.inf, -np.inf, -1e-9):
        for k in (0, ntau // 2, ntau - 1):
            w = v.copy()
            w[k] = bad
            assert np.all(np.isnan(af.fit(w, N, FS)))
    # ntau = 0: the series is too short for one tau (allan.py:32)
    assert af.grid(80, 10.0)[0].size == 0
    assert np.all(np.isnan(af.fit(np.zeros(0), 80, 10.0)))
    assert af.fit_batch(np.zeros((3, 0)), 80, 10.0).shape == (3, 6)
    # all zero: six zeros
    assert np.array_equal(af.fit(np.zeros(ntau), N, FS), np.zeros(6))
    # a zero bin leaves the fit and sets B_min to 0
    w = v.copy()
    w[3] = 0.0
    out, info = af.fit(w, N, FS, detail=True)
    D, b, s, use = af.system(w, *af.grid(N, FS))
    assert D.shape[0] == ntau - 1 and not use[3]
    assert out[5] == 0.0 and np.all(np.isfinite(out))
    # fewer usable bins than terms: only the supports that fit are tried
    w = np.zeros(ntau)
    w[[4, 20]] = v[[4, 20]]
    _, info = af.fit(w, N, FS, detail=True)
    assert bin(info['mask']).count('1') <= 2 and all(bin(m).count('1') <= 2 for m in info['objectives'])
    w = np.zeros(ntau)
    w[10] = 2.5e-7
    out, info = af.fit(w, N, FS, detail=True)
    assert bin(info['mask']).count('1') == 1 and info['objective'] <= 1e-12 * info['W']


@pytest.mark.parametrize('kind', sorted(af.LAWS))
def test_law_envelopes(kind):
    """The oracle on NumPy-generated series of known coefficients stays inside the envelopes the GPU law tests
    use (oracle/allan_fit_np.py LAWS)."""
    rng = np.random.default_rng(100 + sorted(af.LAWS).index(kind))
    c = af.LAWS[kind]
    ratios = [af.fit(oracle_np.allan_var(af.law_series(kind, rng), af.LAW_FS)[0], af.LAW_N, af.LAW_FS)[c['col']]
              / c['truth'] for _ in range(16)]
    ok, got = af.law_check(kind, ratios)
    assert ok, (kind, got, c)


def test_allan_constructor():
    from gnss_ins_sim_b200.allan_analysis import Allan, Hadamard
    assert Allan().output == ['algo_time', 'ad_accel', 'ad_gyro']
    assert Allan(overlapping=True).output == ['algo_time', 'ad_accel', 'ad_gyro']
    assert Allan(fit=True).output == ['algo_time', 'ad_accel', 'ad_gyro', 'noise_accel', 'noise_gyro']
    assert Allan(True, True).fit and Allan(fit=np.bool_(True)).fit and not Allan().fit
    for bad in (1, 0, 'yes', None, 1.0):
        with pytest.raises(TypeError):
            Allan(fit=bad)
    with pytest.raises(TypeError):
        Hadamard(fit=True)
    assert not Hadamard().fit and Hadamard().output == ['algo_time', 'hd_accel', 'hd_gyro']


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def test_c_abi_argument_checks_are_pinned():
    """b2ins_allan_fit_f64 and b2ins_allan_fit_f64_host: each bad argument gives B2INS_ERR_ARG and a pinned
    b2ins_last_error() text before any CUDA call; nseries = 0 returns B2INS_OK; without a device, valid arguments
    reach CUDA (B2INS_ERR_CUDA).  With a device the valid calls are not made: the device entry would launch K13 on
    these host buffers."""
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    ntau = len(af.grid(N, FS)[0])
    var, out = np.ones(4 * ntau), np.zeros(4 * 6)
    good = dict(fs=FS, n=N, ns=4, var=var, ss=ntau, bs=1, out=out)
    too_many = 'too many series for one call'
    cases = [
        (dict(fs=0.0), 'bad fs/n/nseries'), (dict(fs=-1.0), 'bad fs/n/nseries'), (dict(fs=np.inf), 'bad fs/n/nseries'),
        (dict(fs=np.nan), 'bad fs/n/nseries'), (dict(n=-1), 'bad fs/n/nseries'), (dict(ns=-1), 'bad fs/n/nseries'),
        (dict(ss=-1), 'bad strides'), (dict(bs=0), 'bad strides'), (dict(bs=-3), 'bad strides'),
        (dict(var=None), 'null buffer'), (dict(out=None), 'null buffer'),
        (dict(ns=0, var=None, out=None), None), (dict(ns=0, ss=-1), 'bad strides'),
        # one CTA per four series: 2^31 - 1 CTAs at most, so 4 (2^31 - 1) series and not one more
        (dict(ns=4 * (2 ** 31 - 1) + 1), too_many), (dict(ns=2 ** 62), too_many), (dict(ns=2 ** 63 - 1), too_many),
        (dict(n=80, fs=10.0, var=None), 'valid'),           # ntau = 0: var may be null
        ({}, 'valid'),
    ]
    has_device = lib.b2ins_device_count() > 0
    for host in (False, True):
        for change, want in cases:
            if want == 'valid' and has_device:
                continue
            a = dict(good, **change)
            args = [a['fs'], a['n'], a['ns'], _p(a['var']), a['ss'], a['bs'], _p(a['out'])]
            rc = lib.b2ins_allan_fit_f64_host(*args) if host else lib.b2ins_allan_fit_f64(*(args + [None]))
            if want is None:
                assert rc == _lib.OK, (host, change, rc)
            elif want == 'valid':
                assert rc == _lib.ERR_CUDA, (host, change, rc)
            else:
                assert (rc, lib.b2ins_last_error().decode()) == (_lib.ERR_ARG, want), (host, change)


@pytest.mark.parametrize('fit', [False, True])
def test_multi_rank_gather_keeps_curves_and_noise_apart(monkeypatch, fit):
    """Sim's gather of the Allan results of two ranks (uneven shards, 3 + 2 runs): each rank's curves and noise
    terms travel as one row per run, and every rank unpacks all runs' curves and noise terms in run order.  The
    collective is replaced by the concatenation of the rows each rank hands it."""
    from gnss_ins_sim_b200 import sim as simmod
    rng = np.random.default_rng(9)
    L, shards = 7, [(0, 3), (3, 5)]
    curves = rng.standard_normal((5, L, 6))
    noise = rng.standard_normal((5, 6, 6)) if fit else None
    handed = {}
    for r, (lo, hi) in enumerate(shards):
        def record(local, total, r=r):
            handed[r] = local.numpy().copy()
            return np.zeros((total, local.shape[1]))
        monkeypatch.setattr(simmod.dist, 'gather_rows', record)
        simmod._gather_allan(curves[lo:hi], None if noise is None else noise[lo:hi], 5)
    assert [handed[r].shape for r in (0, 1)] == [(3, 6 * L + 36 * fit), (2, 6 * L + 36 * fit)]
    monkeypatch.setattr(simmod.dist, 'gather_rows', lambda local, total: np.concatenate([handed[0], handed[1]]))
    for lo, hi in shards:
        c, z = simmod._gather_allan(curves[lo:hi], None if noise is None else noise[lo:hi], 5)
        assert np.array_equal(c, curves)
        assert (z is None) if not fit else np.array_equal(z, noise)
