"""The device's FP64 primitives (csrc/fastmath64.cuh, mech.cuh's sincos_angle) and its Box-Muller normals,
run on the GPU through the production functions themselves (b2ins_diag_fastmath_f64, b2ins_diag_philox,
b2ins_diag_normal_from_words) and held to the exact reference oracle/fastmath_exact.py: ~2^22 random
arguments per function and domain plus every hard case, in one launch each.

The device forms differ from the host's: rcp_nr / div_nr / sqrt_nr / rsqrt_nr are hardware seeds plus
Newton steps (IEEE operations on the host), and nvcc contracts five multiply/add pairs of log_unit into
DFMAs, so log_unit is held to its bound only.  sincos_bounded, sincos_angle and sincospi_2u have no
contractible pairs and must equal the host build (tests/test_cpu_fastmath.py) bit for bit.  The worst error
per function and domain, and where it occurs, is printed."""
import ctypes

import numpy as np
import pytest

import fastmath_exact as fx
from test_cpu_fastmath import FM, PHILOX_KAT, build_host_lib, host_eval, oracle_philox, philox_ctr_keys

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not fx.have_long_double(),
                                 reason='np.longdouble has no 64-bit significand here: no exact reference')]
torch = pytest.importorskip('torch')

N = 1 << 22
WORST = {}                       # (function, domain) -> (worst, unit, argument)


@pytest.fixture(scope='module')
def lib():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import _lib
    yield _lib
    if WORST:
        print('\nworst device error per function and domain:')
        for (fn, dom), (v, unit, arg) in sorted(WORST.items()):
            print('  %-15s %-24s %.4g %-6s at %r' % (fn, dom, v, unit, arg))


@pytest.fixture(scope='module')
def host(tmp_path_factory):
    return build_host_lib(tmp_path_factory.mktemp('fastmath_host'))


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def dev_eval(lib, name, a, b=None):
    """name on the device over a (and b), one launch: one array, or (sin, cos)."""
    ta = torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()
    tb = None if b is None else torch.from_numpy(np.ascontiguousarray(b, dtype=np.float64)).cuda()
    o0 = torch.empty_like(ta)
    o1 = torch.empty_like(ta) if name.startswith('sincos') else None
    lib.check(lib.load().b2ins_diag_fastmath_f64(FM[name], ta.numel(), _p(ta), _p(tb), _p(o0), _p(o1)))
    return (o0.cpu().numpy(), o1.cpu().numpy()) if o1 is not None else o0.cpu().numpy()


def record(fn, dom, err, args, unit):
    i = int(np.argmax(err))
    WORST[(fn, dom)] = (float(err[i]), unit, args[i] if not isinstance(args, tuple) else
                        tuple(float(a[i]) for a in args))
    return float(err[i])


# ---- the elementary functions -------------------------------------------------------------------------
@pytest.mark.parametrize('dom', ['uniform', 'pi'])
def test_sincos_bounded(lib, host, dom):
    x = fx.sincos_args(N // 2, 1)
    if dom == 'pi':
        x = np.concatenate([np.random.default_rng(21).uniform(-np.pi, np.pi, N), x[np.abs(x) <= np.pi]])
    s, c = dev_eval(lib, 'sincos_bounded', x)
    hs, hc = host_eval(host, 'sincos_bounded', x)
    assert np.array_equal(s, hs) and np.array_equal(c, hc), 'device and host builds differ'
    rs, rc = fx.sincos_ref(x)
    k = fx.sincos_excess(x, s, c, rs, rc)
    w = record('sincos_bounded', '|x|<=64 ' + dom, k, x, 'K')
    record('sincos_bounded', '|x|<=64 %s (ulp)' % dom, np.maximum(fx.ulp_err(s, rs), fx.ulp_err(c, rc)), x, 'ulp')
    assert w <= fx.SINCOS_K, 'K %.4f at %r' % (w, x[np.argmax(k)])


def test_sincos_angle(lib, host):
    x = fx.sincos_angle_args(N, 2)
    s, c = dev_eval(lib, 'sincos_angle', x)
    hs, hc = host_eval(host, 'sincos_angle', x)
    assert np.array_equal(s, hs) and np.array_equal(c, hc), 'device and host builds differ'
    rs, rc = fx.sincos_ref(x)
    k = fx.sincos_excess(x, s, c, rs, rc)
    w = record('sincos_angle', '64<|x|<=1e6', k, x, 'K')
    q = fx.quadrant(x)
    d = np.maximum(np.abs(s.astype(fx.LD) - rs), np.abs(c.astype(fx.LD) - rc)).astype(np.float64)
    record('sincos_angle', '64<|x|<=1e6 (abs)', d, x, 'abs')
    assert (d <= fx.SINCOS_ANGLE_K * 2.0 ** -52 + q * fx.PIO2_SPLIT_ERR).all()
    assert w <= fx.SINCOS_ANGLE_K, 'K %.4f at %r' % (w, x[np.argmax(k)])


def test_sincos_angle_specials(lib):
    x = fx.sincos_angle_specials()
    s, c = dev_eval(lib, 'sincos_angle', x)
    big = np.isfinite(x) & (np.abs(x) > fx.ANGLE_LIMIT)
    assert (s[big] == 0).all() and (c[big] == 1).all(), 'beyond 1e6: exactly (0, 1)'
    bad = ~np.isfinite(x)
    assert np.isnan(s[bad]).all() and np.isnan(c[bad]).all(), '+-inf and NaN: NaN'
    zero = x == 0
    assert (s[zero] == 0).all() and (c[zero] == 1).all()


def test_sincospi_2u(lib, host):
    x = fx.sincospi_args(N, 3)
    s, c = dev_eval(lib, 'sincospi_2u', x)
    hs, hc = host_eval(host, 'sincospi_2u', x)
    assert np.array_equal(s, hs) and np.array_equal(c, hc), 'device and host builds differ'
    rs, rc = fx.sincospi_ref(x)
    d = np.maximum(np.abs(s.astype(fx.LD) - rs), np.abs(c.astype(fx.LD) - rc)).astype(np.float64)
    w = record('sincospi_2u', 'x = 2m 2^-52', d, x, 'abs')
    assert w <= fx.SINCOSPI_ABS
    s, c = dev_eval(lib, 'sincospi_2u', np.array([0.0, 0.5, 1.0, 1.5]))
    assert list(s) == [0.0, 1.0, 0.0, -1.0] and list(c) == [1.0, 0.0, -1.0, 0.0]


def test_log_unit(lib):
    x = fx.log_args(N // 2, 4)
    e = fx.ulp_err(dev_eval(lib, 'log_unit', x), fx.log_ref(x))
    w = record('log_unit', '[2^-52, 1]', e, x, 'ulp')
    assert w <= fx.LOG_ULP
    assert dev_eval(lib, 'log_unit', np.array([1.0]))[0] == 0.0


def test_sqrt_nr(lib):
    x = fx.sqrt_args(N // 2, 7)
    got = dev_eval(lib, 'sqrt_nr', x)
    e = fx.sqrt_err(x, got)
    w = record('sqrt_nr', '[0, 72.1]', e, x, 'ulp')
    assert w <= fx.SQRT_ULP
    z = dev_eval(lib, 'sqrt_nr', np.array([0.0, -0.0]))
    assert (z == 0).all()


def test_rsqrt_nr(lib):
    x = fx.rsqrt_args(N, 8)
    e = fx.ulp_err(dev_eval(lib, 'rsqrt_nr', x), fx.rsqrt_ref(x))
    assert record('rsqrt_nr', 'q in [0.9933, 1]', e, x, 'ulp') <= fx.RSQRT_ULP


def test_rcp_nr(lib):
    x = fx.rcp_args(N // 3, 5)
    e = fx.rcp_err(x, dev_eval(lib, 'rcp_nr', x))
    assert record('rcp_nr', 'cos, radii', e, x, 'ulp') <= fx.RCP_ULP


def test_div_nr(lib):
    a, b = fx.div_args(N // 3, 6)
    e = fx.div_err(a, b, dev_eval(lib, 'div_nr', a, b))
    assert record('div_nr', 'sigma/R, f/(2+f)', e, (a, b), 'ulp') <= fx.DIV_ULP


# ---- Philox and Box-Muller ----------------------------------------------------------------------------
def dev_philox(lib, ck):
    t = torch.from_numpy(np.ascontiguousarray(ck, dtype=np.uint32).view(np.int32)).cuda()
    out = torch.empty((ck.shape[0], 4), dtype=torch.int32, device='cuda')
    lib.check(lib.load().b2ins_diag_philox(ck.shape[0], _p(t), _p(out)))
    return out.cpu().numpy().view(np.uint32)


def dev_normals(lib, words):
    t = torch.from_numpy(np.ascontiguousarray(words, dtype=np.uint32).view(np.int32)).cuda()
    z = torch.empty((words.shape[0], 2), dtype=torch.float64, device='cuda')
    lib.check(lib.load().b2ins_diag_normal_from_words(words.shape[0], _p(t), _p(z)))
    return z.cpu().numpy()


def test_philox_bit_exact(lib):
    ck = philox_ctr_keys()
    words = dev_philox(lib, ck)
    assert np.array_equal(words, oracle_philox(ck))
    for c, k, want in PHILOX_KAT:
        got = dev_philox(lib, np.array([c + k], dtype=np.uint32))[0]
        assert tuple(int(w) for w in got) == want


def _check_normals(z, words, what):
    z0, z1, r = fx.box_muller_ref(words)
    B = fx.box_muller_bound()
    d = np.maximum(np.abs(z[:, 0].astype(fx.LD) - z0), np.abs(z[:, 1].astype(fx.LD) - z1))
    with np.errstate(divide='ignore', invalid='ignore'):
        rel = np.where(r > 0, d / (r * fx.LD(2.0 ** -52)), np.where(d == 0, 0, np.inf)).astype(np.float64)
    m1 = ((words[:, 1].astype(np.uint64) << np.uint64(32)) | words[:, 0]) >> np.uint64(12)
    record('normal_from_words', what, rel, m1, 'r*2^-52')
    assert rel.max() <= B, '%s: |z - z*| = %.3f r* 2^-52 > B = %.3f' % (what, rel.max(), B)


def test_box_muller_edges(lib):
    top = (1 << 52) - 1
    m2 = np.concatenate([[0, 1 << 50, 1 << 51, 3 << 50], (3 << 50) + np.arange(-64, 65), np.arange(0, 65),
                         (1 << 50) + np.arange(-64, 65), (1 << 51) + np.arange(-64, 65), top - np.arange(0, 64)])
    m1 = np.array([0, 1, 2, top, top - 1, 1 << 51, 12345], dtype=np.uint64)
    mm1, mm2 = np.meshgrid(m1, m2.astype(np.uint64), indexing='ij')
    words = fx.words_from_m(mm1.ravel(), mm2.ravel())
    z = dev_normals(lib, words)
    _check_normals(z, words, 'edges')
    # m1 = 0: u1 = 1, r = 0 through sqrt_nr's zero select, z = +-0 exactly
    zero = mm1.ravel() == 0
    assert (z[zero] == 0).all()
    # quadrant points: (r, 0), (0, r), (-r, 0), (0, -r) exactly
    _, _, r = fx.box_muller_ref(words)
    for m, (c, s) in ((0, (1, 0)), (1 << 50, (0, 1)), (1 << 51, (-1, 0)), (3 << 50, (0, -1))):
        at = (mm2.ravel() == m) & ~zero
        got_r = z[at, 0] if c else z[at, 1]
        assert (z[at, 1 if c else 0] == 0).all(), m
        assert (np.sign(got_r) == (c or s)).all(), m
        # the r the device computes: its own sqrt_nr(-2 log_unit(u1)), exact in the other component
        assert (fx.ulp_err(np.abs(got_r), r[at]) <= fx.LOG_ULP / 2 + fx.SQRT_ULP + 1e-3).all(), m
    # r at u1 = 2^-52 is sqrt(104 ln 2) = 8.49
    far = mm1.ravel() == top
    assert np.abs(np.hypot(z[far, 0], z[far, 1]) - 8.4909) .max() < 1e-3


def test_box_muller_ignores_the_discarded_bits(lib):
    rng = np.random.default_rng(31)
    words = rng.integers(0, 1 << 32, (4096, 4), dtype=np.uint64).astype(np.uint32)
    flipped = words.copy()
    flipped[:, 0] ^= rng.integers(1, 1 << 12, 4096, dtype=np.uint64).astype(np.uint32)
    flipped[:, 2] ^= rng.integers(1, 1 << 12, 4096, dtype=np.uint64).astype(np.uint32)
    clear = words & np.array([0xFFFFF000, 0xFFFFFFFF, 0xFFFFF000, 0xFFFFFFFF], dtype=np.uint32)
    a, b, c = dev_normals(lib, words), dev_normals(lib, flipped), dev_normals(lib, clear)
    assert np.array_equal(a, b) and np.array_equal(a, c)


def test_box_muller_random_words(lib):
    words = np.random.default_rng(32).integers(0, 1 << 32, (N, 4), dtype=np.uint64).astype(np.uint32)
    _check_normals(dev_normals(lib, words), words, 'random words')


def test_normals_are_k1s(lib):
    """philox + normal_from_words on (t, draw, run, seed) equal K1's dumped normals bit for bit, with a
    seed and run ids whose high words are set."""
    from gnss_ins_sim_b200 import engine
    seed = (0xFEDCBA98 << 32) | 0x76543210
    run0 = (1 << 32) - 2                      # runs straddle the run id's high word
    R, n = 4, 257
    zero3 = np.zeros(3)
    ge = {'b': zero3, 'b_drift': zero3 + 1e-5, 'b_corr': np.full(3, 100.0), 'arw': zero3 + 1e-4}
    ae = {'b': zero3, 'b_drift': zero3 + 1e-4, 'b_corr': np.full(3, 100.0), 'vrw': zero3 + 1e-3}
    ref = torch.zeros((n, 3), dtype=torch.float64, device='cuda')
    _, _, z = engine.imu_noise(100.0, R, ref, ref, ge, ae, seed, run0, dump_z=True)
    z = z.cpu().numpy()
    runs = run0 + np.arange(R, dtype=np.uint64)
    t, draw, run = np.meshgrid(np.arange(n, dtype=np.uint64), np.arange(6, dtype=np.uint64), runs, indexing='ij')
    ck = np.stack([t, draw, run & np.uint64(0xFFFFFFFF), run >> np.uint64(32),
                   np.full_like(t, seed & 0xFFFFFFFF), np.full_like(t, seed >> 32)], -1).reshape(-1, 6)
    zz = dev_normals(lib, dev_philox(lib, ck.astype(np.uint32))).reshape(n, 6, R, 2)
    # K1's dump: (acc z0[3], acc z1[3], gyro z0[3], gyro z1[3]); draws 0..2 accel, 3..5 gyro
    want = np.concatenate([zz[:, 0:3, :, 0], zz[:, 0:3, :, 1], zz[:, 3:6, :, 0], zz[:, 3:6, :, 1]], axis=1)
    assert np.array_equal(z, want.transpose(2, 0, 1))
