"""The FP64 primitives of csrc/fastmath64.cuh (and mech.cuh's sincos_angle) compiled for the HOST
(tools/fastmath_host.cu, nvcc's host pass) and held to the exact reference oracle/fastmath_exact.py on the
domains and hard cases tests/test_gpu_fastmath.py holds the device to; the reference itself held to mpmath;
the device's constant table held to the literals the host compiles; and the noise generator's Philox
(the oracle's, which the device matches bit for bit) held to the Random123 known-answer vectors and to
cuRAND's independent curand_Philox4x32_10.  Needs nvcc (host pass only); no GPU.

On the host, rcp_nr, div_nr, sqrt_nr and rsqrt_nr are IEEE 1/x, a/b and sqrt, and log_unit has no
contracted multiply-adds: their device forms are measured by the GPU test only."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import fastmath_exact as fx
import oracle_np as onp

SRC = os.path.join(ROOT, 'tools', 'fastmath_host.cu')
HEADER = os.path.join(ROOT, 'gnss_ins_sim_b200', 'csrc', 'fastmath64.cuh')
N = 1 << 20                     # random arguments per domain (the GPU test uses 2^22)
FM = {name: i for i, name in enumerate(('rcp_nr', 'div_nr', 'sqrt_nr', 'rsqrt_nr', 'sincos_bounded',
                                        'sincos_angle', 'sincospi_2u', 'log_unit'))}

# Random123 known-answer vectors of Philox4x32-10: (counter, key) -> words
PHILOX_KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]

pytestmark = pytest.mark.skipif(not fx.have_long_double(),
                                reason='np.longdouble has no 64-bit significand here: no exact reference')


def build_host_lib(out_dir):
    """Compile tools/fastmath_host.cu into out_dir; returns the loaded library (or skips without nvcc)."""
    nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
    if not os.path.exists(nvcc):
        pytest.skip('nvcc not available')
    lib_path = os.path.join(str(out_dir), 'libfastmath_host.so')
    subprocess.run([nvcc, '-O2', '-std=c++17', '-shared', '-Xcompiler', '-fPIC', '-DB2INS_HOST_TEST',
                    '-Wno-deprecated-gpu-targets', '-o', lib_path, SRC], check=True, capture_output=True)
    lib = ctypes.CDLL(lib_path)
    P = ctypes.c_void_p
    lib.fastmath_host.argtypes = [ctypes.c_int, ctypes.c_int64, P, P, P, P]
    lib.philox_curand.argtypes = [ctypes.c_int64, P, P]
    return lib


def host_eval(lib, name, a, b=None):
    """name's host form on a (and b): one array, or (sin, cos)."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = None if b is None else np.ascontiguousarray(b, dtype=np.float64)
    pair = name.startswith('sincos')
    o0 = np.empty_like(a)
    o1 = np.empty_like(a) if pair else None
    p = lambda x: None if x is None else x.ctypes.data_as(ctypes.c_void_p)
    lib.fastmath_host(FM[name], a.size, p(a), p(b), p(o0), p(o1))
    return (o0, o1) if pair else o0


def philox_ctr_keys(seed=5):
    """[n, 6] counters and keys: every word from {0, 1, 0x7FFFFFFF, 0xFFFFFFFE, 0xFFFFFFFF} in turn, the
    draws K7 makes at t = 0xFFFFFFFE and the phase draws at t = 0xFFFFFFFF, seeds and run ids with
    non-zero high words, random rows, and the known-answer rows."""
    rng = np.random.default_rng(seed)
    special = np.array([0, 1, 0x7FFFFFFF, 0xFFFFFFFE, 0xFFFFFFFF], dtype=np.uint64)
    rows = []
    base = rng.integers(0, 1 << 32, (len(special) * 6, 6), dtype=np.uint64)
    for w in range(6):
        for j, v in enumerate(special):
            r = base[w * len(special) + j].copy()
            r[w] = v
            rows.append(r)
    grid = np.array(np.meshgrid(special, special, indexing='ij')).reshape(2, -1).T
    for t in (0, 1, 0xFFFFFFFE, 0xFFFFFFFF):              # (t, draw) x (run_hi, seed_hi) corners
        for d in (0, 3, 9, 16, 24):
            for rh, sh in grid:
                rows.append(np.array([t, d, 0x89ABCDEF, rh, 0x01234567, sh], dtype=np.uint64))
    seed64 = (1 << 63) + 12345
    for run in (0, 1, (1 << 32) - 1, 1 << 32, (1 << 32) + 7, (1 << 40) + 3):
        for t in (0, 99, 0xFFFFFFFE, 0xFFFFFFFF):
            rows.append(np.array([t, 3, run & 0xFFFFFFFF, run >> 32, seed64 & 0xFFFFFFFF, seed64 >> 32],
                                 dtype=np.uint64))
    rows += [np.array(c + k, dtype=np.uint64) for c, k, _ in PHILOX_KAT]
    rows = np.array(rows, dtype=np.uint64)
    return np.concatenate([rows, rng.integers(0, 1 << 32, (4096, 6), dtype=np.uint64)]).astype(np.uint32)


def oracle_philox(ck):
    ck = np.asarray(ck, dtype=np.uint64)
    out = [onp.philox4x32_10(ck[i, 0], ck[i, 1], ck[i, 2], ck[i, 3], int(ck[i, 4]), int(ck[i, 5]))
           for i in range(ck.shape[0])]
    return np.array([[int(w) for w in o] for o in out], dtype=np.uint32)


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp('fastmath_host'))


# ---- the host forms against the exact reference ---------------------------------------------------------
def test_sincos_bounded_host(host):
    x = fx.sincos_args(N, 1)
    s, c = host_eval(host, 'sincos_bounded', x)
    rs, rc = fx.sincos_ref(x)
    k = fx.sincos_excess(x, s, c, rs, rc)
    assert k.max() <= fx.SINCOS_K, 'K %.4f at x = %r' % (k.max(), x[k.argmax()])


def test_sincos_angle_host(host):
    x = fx.sincos_angle_args(N, 2)
    s, c = host_eval(host, 'sincos_angle', x)
    rs, rc = fx.sincos_ref(x)
    k = fx.sincos_excess(x, s, c, rs, rc)
    assert k.max() <= fx.SINCOS_ANGLE_K, 'K %.4f at x = %r' % (k.max(), x[k.argmax()])


def test_sincos_angle_host_specials(host):
    x = fx.sincos_angle_specials()
    s, c = host_eval(host, 'sincos_angle', x)
    big = np.isfinite(x) & (np.abs(x) > fx.ANGLE_LIMIT)
    assert (s[big] == 0).all() and (c[big] == 1).all()
    bad = ~np.isfinite(x)
    assert np.isnan(s[bad]).all() and np.isnan(c[bad]).all()
    zero = x == 0                     # sin(-0) is +0 here (r z ps + r rounds -0 + -0 ps up); only the value counts
    assert (s[zero] == 0).all() and (c[zero] == 1).all()
    lim = np.abs(x) == fx.ANGLE_LIMIT                         # the last angle still taken as itself
    rs, rc = fx.sincos_ref(x[lim])
    assert (fx.ulp_err(s[lim], rs) <= fx.SINCOS_ANGLE_K).all() and (fx.ulp_err(c[lim], rc) <= fx.SINCOS_ANGLE_K).all()


def test_sincospi_2u_host(host):
    x = fx.sincospi_args(N, 3)
    s, c = host_eval(host, 'sincospi_2u', x)
    rs, rc = fx.sincospi_ref(x)
    d = np.maximum(np.abs(s.astype(fx.LD) - rs), np.abs(c.astype(fx.LD) - rc)).astype(np.float64)
    assert d.max() <= fx.SINCOSPI_ABS, '%.3e at x = %r' % (d.max(), x[d.argmax()])
    s, c = host_eval(host, 'sincospi_2u', np.array([0.0, 0.5, 1.0, 1.5]))
    assert list(s) == [0.0, 1.0, 0.0, -1.0] and list(c) == [1.0, 0.0, -1.0, 0.0]


def test_log_unit_host(host):
    x = fx.log_args(N, 4)
    e = fx.ulp_err(host_eval(host, 'log_unit', x), fx.log_ref(x))
    assert e.max() <= fx.LOG_ULP, '%.4f ulp at x = %r' % (e.max(), x[e.argmax()])
    assert host_eval(host, 'log_unit', np.array([1.0]))[0] == 0.0


def test_ieee_forms_host(host):
    """On the host the Newton forms are the IEEE operations: correctly rounded, so the exact-error
    functions the GPU test relies on give at most half an ulp here, and sqrt(0) is 0."""
    x = fx.rcp_args(N // 4, 5)
    assert fx.rcp_err(x, host_eval(host, 'rcp_nr', x)).max() <= 0.5
    a, b = fx.div_args(N // 4, 6)
    assert fx.div_err(a, b, host_eval(host, 'div_nr', a, b)).max() <= 0.5
    x = fx.sqrt_args(N // 4, 7)
    assert fx.sqrt_err(x, host_eval(host, 'sqrt_nr', x)).max() <= 0.5
    x = fx.rsqrt_args(N // 4, 8)
    assert fx.ulp_err(host_eval(host, 'rsqrt_nr', x), fx.rsqrt_ref(x)).max() <= fx.RSQRT_ULP


def test_exact_errors_resolve_the_sqrt_bound():
    """The exact errors see what long double cannot: the neighbour of a correctly rounded sqrt is 1 -+ e of
    an ulp off where the rounded one is e; the error functions report the exact value at their maximum and
    the long-double estimate (good to EXACT_SLACK) elsewhere; and rcp / div count the same way."""
    rng = np.random.default_rng(9)
    x = rng.uniform(1e-3, 72.1, 200)
    cr = np.sqrt(x)
    nb = np.nextafter(cr, np.inf)
    e_cr = np.array([fx._sqrt_frac_err(float(a), float(s)) for a, s in zip(x, cr)])
    e_nb = np.array([fx._sqrt_frac_err(float(a), float(s)) for a, s in zip(x, nb)])
    assert (e_cr <= 0.5).all() and (np.abs(fx.sqrt_err(x, cr) - e_cr) <= fx.EXACT_SLACK).all()
    assert ((e_nb > 0.5) & (e_nb < 1.5)).all()
    assert (np.minimum(np.abs(e_nb - (1 - e_cr)), np.abs(e_nb - (1 + e_cr))) <= 1e-12).all()
    got = fx.sqrt_err(x, nb)
    assert np.abs(got - e_nb).max() <= fx.EXACT_SLACK and got.max() == e_nb.max()
    assert fx.sqrt_err(np.array([0.0, 0.0]), np.array([0.0, 1e-300]))[1] == np.inf
    y = rng.uniform(0.5, 2.0, 100)
    assert (fx.rcp_err(y, np.nextafter(1.0 / y, np.inf)) > 0.5).all()
    assert (fx.div_err(y, 3.0 * y, np.nextafter(y / (3.0 * y), 0.0)) > 0.5).all()


# ---- the reference against mpmath ---------------------------------------------------------------------
def test_long_double_reference_against_mpmath():
    mpmath = pytest.importorskip('mpmath')
    mpmath.mp.dps = 100
    rng = np.random.default_rng(10)
    pick = lambda a, k: a[rng.choice(a.size, min(k, a.size), replace=False)]
    tol = 2.0 ** -62

    def rel(ld, exact):
        d = abs(mpmath.mpf(fx.ld_fraction(ld).numerator) / fx.ld_fraction(ld).denominator - exact)
        return float(d / abs(exact)) if exact != 0 else float(d)

    x = np.concatenate([pick(fx.halfpi_multiples(fx.ANGLE_LIMIT), 200), pick(fx.odd_quarterpi_multiples(), 50),
                        pick(fx.sincos_angle_args(1000, 11), 50)])
    rs, rc = fx.sincos_ref(x)
    for i in range(x.size):
        m = mpmath.mpf(float(x[i]))
        assert rel(rs[i], mpmath.sin(m)) <= tol and rel(rc[i], mpmath.cos(m)) <= tol, x[i]
    x = pick(fx.log_hard_cases(), 200)
    r = fx.log_ref(x)
    for i in range(x.size):
        if x[i] != 1.0:
            assert rel(r[i], mpmath.log(mpmath.mpf(float(x[i])))) <= tol, x[i]
    x = pick(fx.sincospi_args(1000, 12), 100)
    rs, rc = fx.sincospi_ref(x)
    for i in range(x.size):
        a = mpmath.pi * mpmath.mpf(float(x[i]))
        assert rel(rs[i], mpmath.sin(a)) <= 4 * tol and rel(rc[i], mpmath.cos(a)) <= 4 * tol, x[i]
    words = fx.words_from_m(np.array([1, 2, 12345, (1 << 52) - 1, 1 << 51], dtype=np.uint64), np.uint64(1 << 49))
    _, _, r = fx.box_muller_ref(words)
    m1 = [1, 2, 12345, (1 << 52) - 1, 1 << 51]
    for i, m in enumerate(m1):
        exact = mpmath.sqrt(-2 * mpmath.log(1 - mpmath.mpf(m) / 2 ** 52))
        assert rel(r[i], exact) <= tol, m
    split = abs(mpmath.pi / 2 - (mpmath.mpf(fx.PIO2_1) + mpmath.mpf(fx.PIO2_2) + mpmath.mpf(fx.PIO2_3)))
    assert abs(fx.PIO2_SPLIT_ERR - float(split)) <= 1e-6 * float(split)


def test_hard_case_generators():
    x = fx.halfpi_multiples(fx.ANGLE_LIMIT)
    assert x.size == 1 + 2 * 9 * 636619 and np.abs(x).max() <= fx.ANGLE_LIMIT
    q = fx.quadrant(x)
    assert q.max() == 636619
    x = fx.odd_quarterpi_multiples()
    assert np.abs(x).max() <= 64.0 and x.size == 2 * 9 * 41
    x = fx.log_hard_cases()
    assert x.min() == 2.0 ** -52 and x.max() == 1.0
    near_sqrt2 = np.ldexp(math.sqrt(2.0), -1)
    assert (np.abs(x - near_sqrt2) <= 8 * np.spacing(near_sqrt2)).sum() == 17


# ---- the device's constant table ------------------------------------------------------------------------
def test_constant_table_matches_the_literals():
    """The device reads B2K(i, lit) from kB2Const[i], the host compiles lit: both must be the same double."""
    src = open(HEADER).read()
    table = re.search(r'kB2Const\[(\d+)\]\s*=\s*\{([^}]*)\}', src, re.S)
    entries = [float(v) for v in table.group(2).replace('\n', ' ').split(',') if v.strip()]
    assert len(entries) == int(table.group(1))
    uses = re.findall(r'B2K\((\d+),\s*([-+0-9.eE]+)\)', src)
    assert len({int(i) for i, _ in uses}) >= 26 and all(int(i) < len(entries) for i, _ in uses)
    for i, lit in uses:
        a, b = np.float64(float(lit)), np.float64(entries[int(i)])
        assert a.view(np.uint64) == b.view(np.uint64), 'B2K(%s, %s) != kB2Const[%s] = %r' % (i, lit, i, entries[int(i)])
    assert fx.PIO2_1 == entries[13] and fx.PIO2_2 == entries[14] and fx.PIO2_3 == entries[15]


# ---- Philox -------------------------------------------------------------------------------------------
def test_philox_known_answers():
    for c, k, want in PHILOX_KAT:
        got = onp.philox4x32_10(*c, *k)
        assert tuple(int(w) for w in got) == want


def test_philox_matches_curand(host):
    ck = philox_ctr_keys()
    words = np.empty((ck.shape[0], 4), dtype=np.uint32)
    host.philox_curand(ck.shape[0], ck.ctypes.data_as(ctypes.c_void_p), words.ctypes.data_as(ctypes.c_void_p))
    assert np.array_equal(words, oracle_philox(ck))
    kat = {tuple(int(v) for v in r[:6]): tuple(int(v) for v in w) for r, w in zip(ck, words)}
    for c, k, want in PHILOX_KAT:
        assert kat[c + k] == want
