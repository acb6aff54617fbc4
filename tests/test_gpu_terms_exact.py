"""The IEEE Std 952 terms and the run-to-run errors of K1 and K9 (the _ex, _rx and _ex_rx forms) held to the exact
reference of oracle/terms_exact.py, with no free tolerance.

An IMU with only one term set and b = w = wd = 0 stores that term alone at every sample (plus ref where a case
needs one); the draws are the device's own -- uniform01 is integer arithmetic, the walk's drive normals come from
b2ins_diag_philox + b2ins_diag_normal_from_words (tests/test_gpu_fastmath.py shows them K1's), the run-error table
from engine.imu_run_errors.

Quantisation, ramp, run errors: bit for bit.  terms_sample rounds e[t+1] = q (u - 1/2), e[t+1] - e[t], the division
by dt, t dt and R (t dt), exactly as the reference; with one term per channel the others add exact zeros, and a
fused R (t dt) + qr is fl(R (t dt)) when qr = 0 and qr when R = 0.  run_err_add is three fmas and one add, which
terms_exact.run_err_sample emulates exactly.  Quantisation and ramp channels may sit beside walk channels: the
branches are per channel.

Walk: |w^_t - w_t| <= C_walk u Psi_t / (1 - C_walk u), Psi_t = sum_{s<t} (|k z_s| + |w_{s+1}|), derived as
test_gpu_gm_drift.py derives C_K1 (every rounding is of a zero-state partial of the drives it holds, or of a walk
value at some sample), by K1's association order for the walk's channels:
  the fma that takes k z_s (1), the thread's serial stretch (kNoisePer = 7 fmas), the 5-level warp scan (5), <= 3
  warp fmas + the lane's fma + S or the tile carry (5), the add of the terms into the measurement and the add of
  S_walk into the stage (2):  C_walk = 20.
No power factors: the walk's A = 1 is exact in every product (C_K1 = 916 is 896 of them).  With time segments the
carry chain adds one fma per segment end, pow(1, L) = 1 and 1 * c being exact, and pass 1 keeps every drive (the
walk never decays, so pass1_len = seg_len): C_walk_seg = 21.

Everything at once (Gauss-Markov, white, all three terms, run errors, a non-zero reference): within
terms_exact.assemble's bound of the exact sum of the device-drawn components, gamma_19 of their magnitudes plus
the drift's C_K1 and the walk's C_walk bounds.  A term added twice or left out is off by that term, far outside.

K9 is held to K1's series of the same call in every new form: end_err bit for bit (K9 rounds the stage with an
explicit fma, K1 by contraction), proc_stats to stats_exact within the reducer's DEPTH_K9 chains.  Non-finite
references: with run errors set, a NaN in one reference column makes all three channels of that sensor NaN at
that sample (S[c][j] NaN is NaN for S[c][j] = 0 too), as NumPy's ref + b + S @ ref does; the other sensor, and
a launch without the bad value, are unchanged bit for bit.

The worst err / bound per generator is printed at the end of the module."""
import ctypes

import numpy as np
import pytest

import gm_exact as ge
import stats_exact as sx
import terms_exact as tx
from test_gpu_gm_drift import C_K1
from test_gpu_stats_edges import DEPTH_K9, _check

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

U = 2.0 ** -53
FS = 100.0
DT = 1.0 / FS
SEED = (0x0123ABCD << 32) | 0x89ABCDEF
R0 = 2 ** 32 - 2                      # the runs straddle the run id's high word
C_WALK = 1 + 7 + 5 + 5 + 2
C_WALK_SEG = C_WALK + 1
WORST = {}
NS = [1, 2, 7, 8, 895, 896, 897, 1793, 5041]

# one sensor's run errors with no turn-on bias: with ref = 0 they add exact zeros, so K1-ex-rx stores the terms alone
SF_ONLY = {'sf': np.array([3e-3, 1e-3, 2e-3]), 'ma': 2e-3 * (1.0 - np.eye(3))}
RUN_G = {'b_std': np.array([1e-4, 2e-4, 5e-5]), 'sf': np.array([1e-3, 0.0, 5e-4]),
         'ma': np.array([[0.0, 2e-3, 0.0], [3e-3, 0.0, 4e-3], [5e-4, 6e-3, 0.0]])}
RUN_A = {'b_std': np.array([1e-2, 3e-2, 2e-2]), 'sf': np.array([3e-3, 1e-3, 2e-3]), 'ma': 2e-3 * (1.0 - np.eye(3))}
# one term per channel: every channel's sample is that term alone
TERM_CASES = {
    'q': ({'q': np.array([2e-5, 0.0, 3e-5])}, {'q': np.array([0.0, 2e-3, 5e-4])}),
    'rr': ({'rr': np.array([1e-6, -2e-6, 0.0])}, {'rr': np.array([1e-4, 0.0, -2e-4])}),
    'q|rr': ({'q': np.array([2e-5, 0.0, 0.0]), 'rr': np.array([0.0, -2e-6, 0.0])},
             {'q': np.array([0.0, 0.0, 5e-4]), 'rr': np.array([3e-4, 0.0, 0.0])}),
}


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nIEEE Std 952 terms: worst |generated - exact| / bound per generator: ' +
          ', '.join('%s %.3g' % kv for kv in sorted(WORST.items())))


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _zero(key, **kw):
    return dict({'b': np.zeros(3), 'b_drift': np.zeros(3), 'b_corr': np.full(3, np.inf), key: np.zeros(3)}, **kw)


def _errs(gyro=None, accel=None):
    return _zero('arw', **(gyro or {})), _zero('vrw', **(accel or {}))


def _k1(eng, R, n, ge_, ae_, r0=R0, layout=0, rg=None, ra=None, seed=SEED, dump=False):
    """K1 of the call: meas [R, n, 6] (accel x y z, gyro x y z) run-major, and z_dump if asked."""
    rg = eng.to_device(np.zeros((n, 3)) if rg is None else rg)
    ra = eng.to_device(np.zeros((n, 3)) if ra is None else ra)
    out = eng.imu_noise(FS, R, rg, ra, ge_, ae_, seed, run_offset=r0, layout=layout, dump_z=dump)
    gyro, accel = out[0], out[1]
    if layout == eng.LAYOUT_TIME_MAJOR:
        gyro, accel = gyro.permute(2, 0, 1), accel.permute(2, 0, 1)
    elif layout == eng.LAYOUT_CHANNEL_MAJOR:
        gyro, accel = gyro.permute(0, 2, 1), accel.permute(0, 2, 1)
    meas = torch.cat([accel, gyro], dim=2).cpu().numpy()
    return (meas, out[2].cpu().numpy()) if dump else meas


def _run_ids(R, r0=R0):
    return np.arange(R, dtype=np.uint64) + np.uint64(r0)


def _terms_exact(n, ge_, ae_, run_ids, seed=SEED):
    """Quantisation + ramp of both sensors [R, n, 6], exact (one of them per channel)."""
    out = []
    for sensor, err in ((0, ae_), (1, ge_)):
        q, _, r, dt = tx.coefficients(FS, err)
        x = tx.quant_rate(q, tx.quant_uniforms(n, sensor, seed, run_ids), dt)
        assert not np.any((q != 0.0) & (r != 0.0)), 'one term per channel'
        out.append(x + tx.ramp(r, n, dt)[None])
    return np.concatenate(out, axis=2)


def _walk_normals(eng, n, run_ids, seed=SEED):
    """The walk's drive normals z0 [R, n, 6] (draws 32 + 3 s + c) from the device's Philox and Box-Muller."""
    from gnss_ins_sim_b200 import _lib
    R = len(run_ids)
    t, d, r = np.meshgrid(np.arange(n, dtype=np.uint64), np.arange(32, 38, dtype=np.uint64), run_ids, indexing='ij')
    ck = np.stack([t, d, r & np.uint64(0xFFFFFFFF), r >> np.uint64(32), np.full_like(t, seed & 0xFFFFFFFF),
                   np.full_like(t, seed >> 32)], -1).reshape(-1, 6).astype(np.uint32)
    lib = _lib.load()
    tc = torch.from_numpy(ck.view(np.int32)).cuda()
    words = torch.empty((ck.shape[0], 4), dtype=torch.int32, device='cuda')
    _lib.check(lib.b2ins_diag_philox(ck.shape[0], _p(tc), _p(words)))
    z = torch.empty((ck.shape[0], 2), dtype=torch.float64, device='cuda')
    _lib.check(lib.b2ins_diag_normal_from_words(ck.shape[0], _p(words), _p(z)))
    return z.cpu().numpy()[:, 0].reshape(n, 6, R).transpose(2, 0, 1)


def _walk_exact(eng, n, ge_, ae_, run_ids, seed=SEED):
    z = _walk_normals(eng, n, run_ids, seed)
    _, ka, _, _ = tx.coefficients(FS, ae_)
    _, kg, _, _ = tx.coefficients(FS, ge_)
    da, pa = tx.walk(ka, z[:, :, :3])
    dg, pg = tx.walk(kg, z[:, :, 3:])
    return np.concatenate([da, dg], axis=2), np.concatenate([pa, pg], axis=2)


def _within(got, d, psi, C, key, what, extra=0.0):
    bound = C * U * psi / (1.0 - C * U) + extra
    err = np.abs(got - d)
    bad = ~(err <= bound)
    assert not bad.any(), '%s: %d samples out of bound, worst err %.3e / bound %.3e at %s' % (
        what, bad.sum(), err[bad].max(), bound[bad][np.argmax(err[bad])], np.argwhere(bad)[0].tolist())
    WORST[key] = max(WORST.get(key, 0.0), float(np.max(err / np.where(bound > 0, bound, np.inf), initial=0.0)))


def _same(got, want, what):
    bad = got != want
    assert not bad.any(), '%s: %d samples differ, first at %s: %r != %r' % (
        what, bad.sum(), np.argwhere(bad)[0].tolist(), got[bad][0], want[bad][0])


# ---- quantisation and ramp, bit for bit ------------------------------------------------------------------------
FORMS = {'ex': ({}, {}), 'ex_rx': (SF_ONLY, SF_ONLY)}


@pytest.mark.parametrize('n', NS)
def test_quantisation_and_ramp_bit_for_bit(eng, n):
    R = 1 + n % 4
    for case, (gt, at) in TERM_CASES.items():
        want = _terms_exact(n, gt, at, _run_ids(R))
        for form, (gx, ax) in FORMS.items():
            ge_, ae_ = _errs(dict(gt, **gx), dict(at, **ax))
            _same(_k1(eng, R, n, ge_, ae_), want, 'K1-%s %s n=%d' % (form, case, n))


@pytest.mark.parametrize('layout', [0, 1, 2])
def test_quantisation_and_ramp_every_layout_and_ragged_runs(eng, layout):
    n = 2 * 896 + 13
    gt, at = TERM_CASES['q|rr']
    for R in (1, 5, 37):
        want = _terms_exact(n, gt, at, _run_ids(R, 1000))
        for form, (gx, ax) in FORMS.items():
            ge_, ae_ = _errs(dict(gt, **gx), dict(at, **ax))
            _same(_k1(eng, R, n, ge_, ae_, r0=1000, layout=layout), want, 'K1-%s layout %d R=%d' % (form, layout, R))


# ---- run errors, bit for bit -------------------------------------------------------------------------------------
def _ref(n, seed=5):
    rng = np.random.default_rng(seed)
    return 0.1 * rng.standard_normal((n, 3)), np.array([0.0, 0.0, -9.8]) + 0.1 * rng.standard_normal((n, 3))


@pytest.mark.parametrize('n', [1, 8, 897, 1793])
def test_run_errors_bit_for_bit(eng, n):
    """K1-rx: ref + the fma chain of the device's table; K1-ex-rx with a ramp on one gyro channel: the ramp joins
    before the run errors, fl(fl(ref + ramp) + delta), and the other channels add an exact zero."""
    R = 3
    rg, ra = _ref(n)
    ramp = {'rr': np.array([0.0, 2e-6, 0.0])}
    for form, gt in (('rx', {}), ('ex_rx', ramp)):
        ge_, ae_ = _errs(dict(RUN_G, **gt), RUN_A)
        tab = eng.imu_run_errors(R, ge_, ae_, SEED, run_offset=R0).cpu().numpy()
        rgr = rg + tx.ramp(tx.coefficients(FS, ge_)[2], n, DT)              # fl(ref + fl(R fl(t dt)))
        want = np.concatenate([np.stack([_fma_chain_plus(ra, ra, tab[r, 0]) for r in range(R)]),
                               np.stack([_fma_chain_plus(rgr, rg, tab[r, 1]) for r in range(R)])], axis=2)
        for layout in ((0, 1, 2) if n == 897 else (0,)):
            _same(_k1(eng, R, n, ge_, ae_, layout=layout, rg=rg, ra=ra), want, 'K1-%s n=%d layout %d' % (form, n, layout))


def _fma_chain_plus(m, ref, t):
    """fl(m + delta), delta = the fma chain of table rows t [3, 4] on ref [n, 3]: run_err_add on the measurement m."""
    d = np.broadcast_to(t[None, :, 3], m.shape)
    for j in range(3):
        d = tx.fma_np(t[None, :, j], ref[:, j:j + 1], d)
    return m + d


# ---- the walk, within C_walk -------------------------------------------------------------------------------------
WALK = ({'rrw': np.array([3e-5, 0.0, 5e-5])}, {'rrw': np.array([1e-3, 3e-4, 0.0])})


@pytest.mark.parametrize('n', NS + [20011])
def test_walk_within_its_bound(eng, n):
    R = 3
    gt, at = WALK
    d, psi = _walk_exact(eng, n, gt, at, _run_ids(R))
    for form, (gx, ax) in FORMS.items():
        ge_, ae_ = _errs(dict(gt, **gx), dict(at, **ax))
        got = _k1(eng, R, n, ge_, ae_)
        _within(got, d, psi, C_WALK, 'K1 walk', 'K1-%s walk n=%d' % (form, n))
        assert np.all(got[:, :, [2, 4]] == 0.0) and np.all(got[:, 0] == 0.0)   # k = 0, and w[0] = 0
        # the first thread's stretch (samples 0 .. 6) starts from S = fma(1, 0, 0) = 0: there the sample is the
        # thread's fma chain itself, fma(k, z_{t-1}, ... fma(k, z_0, 0)), bit for bit
        _same(got[:, :7], _first_stretch(eng, min(n, 7), ge_, ae_, _run_ids(R)), 'K1-%s walk, first stretch' % form)


def _first_stretch(eng, n, ge_, ae_, run_ids):
    z = _walk_normals(eng, n, run_ids)
    k = np.concatenate([tx.coefficients(FS, ae_)[1], tx.coefficients(FS, ge_)[1]])
    out = np.zeros_like(z)
    for t in range(1, n):
        out[:, t] = tx.fma_np(k[None], z[:, t - 1], out[:, t - 1])
    return np.where(k[None, None] != 0.0, out, 0.0)


# ---- time segments: 3 runs x 300 000 samples ---------------------------------------------------------------------
SEG_R, SEG_N = 3, 300000
SEG_CASES = {
    # a walk channel in each sensor beside a quantisation and a ramp channel: pass 1 covers whole segments
    'walk': ({'rrw': np.array([0.0, 0.0, 3e-5]), 'q': np.array([2e-5, 0.0, 0.0]), 'rr': np.array([0.0, -2e-6, 0.0])},
             {'rrw': np.array([1e-3, 0.0, 0.0]), 'q': np.array([0.0, 2e-3, 0.0]), 'rr': np.array([0.0, 0.0, 3e-4])},
             np.inf),
    # quantisation and ramp only, and a short correlation time (b_drift = 0: no drift): pass 1 is shortened
    'short': (TERM_CASES['q|rr'][0], TERM_CASES['q|rr'][1], 0.05),
}
_seg_cache = {}


def _seg_errs(case, run=False):
    gt, at, tau = SEG_CASES[case]
    ge_, ae_ = _errs(dict(gt, **(SF_ONLY if run else {})), dict(at, **(SF_ONLY if run else {})))
    ge_['b_corr'] = ae_['b_corr'] = np.full(3, tau)
    return ge_, ae_


def _segmented(eng, case):
    if case not in _seg_cache:
        from gnss_ins_sim_b200 import _lib
        ge_, ae_ = _seg_errs(case)
        plan = _lib.noise_plan(FS, SEG_R, SEG_N, ge_, ae_)
        ids = _run_ids(SEG_R, 4)
        gt, at, _ = SEG_CASES[case]
        walk_ = {k: v for k, v in gt.items() if k == 'rrw'}, {k: v for k, v in at.items() if k == 'rrw'}
        d, psi = _walk_exact(eng, SEG_N, *walk_, ids)
        qr = ({k: v for k, v in gt.items() if k != 'rrw'}, {k: v for k, v in at.items() if k != 'rrw'})
        _seg_cache[case] = plan, _terms_exact(SEG_N, *qr, ids), d, psi
    return _seg_cache[case]


@pytest.mark.parametrize('case', list(SEG_CASES))
def test_segmented_plans(eng, case):
    plan, exact, d, psi = _segmented(eng, case)
    assert plan['nseg'] >= 3, plan
    if case == 'walk':
        assert plan['pass1_len'] == plan['seg_len']
    else:
        assert plan['pass1_len'] < plan['seg_len'] and np.all(plan['gm_b'] == 0.0) and np.all(np.abs(plan['gm_a']) < 1.0)
    walk_ch = psi.max(axis=(0, 1)) > 0
    for run in (False, True):
        ge_, ae_ = _seg_errs(case, run)
        got = _k1(eng, SEG_R, SEG_N, ge_, ae_, r0=4)
        what = 'K1-%s %s' % ('ex_rx' if run else 'ex', case)
        _same(got[:, :, ~walk_ch], exact[:, :, ~walk_ch], what)
        _within(got[:, :, walk_ch], d[:, :, walk_ch], psi[:, :, walk_ch], C_WALK_SEG, 'K1 walk segmented', what)


# ---- everything at once ------------------------------------------------------------------------------------------
def test_everything_at_once_inside_the_assembly_bound(eng):
    """Gauss-Markov (tau 100 s, 0.05 s, white), white noise, all three terms, run errors and a non-zero reference in
    K1-ex-rx, and the same without run errors in K1-ex: every sample within terms_exact.assemble's bound of the exact
    sum of the components the device draws."""
    from gnss_ins_sim_b200 import _lib
    R, n = 3, 1000
    rg, ra = _ref(n)
    terms_g = {'q': np.array([2e-5, 1e-5, 3e-5]), 'rrw': np.array([3e-5, 1e-5, 5e-5]),
               'rr': np.array([1e-6, -2e-6, 3e-7])}
    terms_a = {'q': np.array([1e-3, 2e-3, 5e-4]), 'rrw': np.array([1e-3, 3e-4, 2e-3]),
               'rr': np.array([1e-4, 0.0, -2e-4])}
    base_g = {'b': np.array([1e-4, 0.0, -2e-4]), 'b_drift': np.full(3, 1e-5), 'b_corr': np.array([100.0, np.inf, 0.05]),
              'arw': np.full(3, 1e-4)}
    base_a = {'b': np.array([0.01, 0.0, -0.02]), 'b_drift': np.full(3, 1e-3), 'b_corr': np.array([np.inf, 50.0, 0.05]),
              'vrw': np.full(3, 1e-3)}
    ids = _run_ids(R)
    for run in (False, True):
        ge_ = dict(base_g, **terms_g, **(RUN_G if run else {}))
        ae_ = dict(base_a, **terms_a, **(RUN_A if run else {}))
        got, zd = _k1(eng, R, n, ge_, ae_, rg=rg, ra=ra, dump=True)
        plan = _lib.noise_plan(FS, R, n, ge_, ae_)
        tab = eng.imu_run_errors(R, ge_, ae_, SEED, run_offset=R0).cpu().numpy()
        wd, wpsi = _walk_exact(eng, n, ge_, ae_, ids)
        for s, (ref, err, key, zs) in enumerate(((ra, ae_, 'vrw', slice(0, 6)), (rg, ge_, 'arw', slice(6, 12)))):
            ch = slice(3 * s, 3 * s + 3)
            z0, z1 = zd[:, :, zs][:, :, :3], zd[:, :, zs][:, :, 3:]
            gm, psi = np.zeros((R, n, 3)), np.zeros((R, n, 3))
            for c in range(3):
                if plan['gm_b'][3 * s + c] != 0.0:
                    gm[:, :, c], psi[:, :, c] = ge.drift(np.full(R, plan['gm_a'][3 * s + c]),
                                                         np.full(R, plan['gm_b'][3 * s + c]), z0[:, :, c])
            q, _, r, dt = tx.coefficients(FS, err)
            sens = {'b': err['b'], 'w': err[key] / np.sqrt(1.0 / FS), 'wd': plan['wd'][ch]}
            ex, bound = tx.assemble(ref, sens, z1, z0, gm, psi, wd[:, :, ch], wpsi[:, :, ch],
                                    tx.quant_rate(q, tx.quant_uniforms(n, s, SEED, ids), dt), tx.ramp(r, n, dt),
                                    tab[:, s], C_K1, C_WALK)
            _within(got[:, :, ch], ex, np.ones_like(bound), 0, 'K1 all terms', 'K1 all run=%s sensor %d' % (run, s),
                    extra=bound)


# ---- K9 against K1 of the same call ------------------------------------------------------------------------------
K9_FORMS = {
    'ex': ({'q': np.array([2e-5, 1e-5, 3e-5]), 'rrw': np.array([3e-5, 1e-5, 5e-5]), 'rr': np.array([1e-6, -2e-6, 3e-7])},
           {'q': np.array([1e-3, 0.0, 5e-4]), 'rrw': np.array([1e-3, 3e-4, 0.0]), 'rr': np.array([1e-4, 0.0, -2e-4])}),
    'rx': (RUN_G, RUN_A),
}
K9_FORMS['ex_rx'] = (dict(K9_FORMS['ex'][0], **RUN_G), dict(K9_FORMS['ex'][1], **RUN_A))
MID_G = {'b': np.array([1e-5, -2e-5, 3e-6]), 'b_drift': np.full(3, 3.5 * np.pi / 180 / 3600),
         'b_corr': np.array([100.0, np.inf, 0.05]), 'arw': np.full(3, 0.25 * np.pi / 180 / 60)}
MID_A = {'b': np.array([2e-3, -1e-3, 5e-4]), 'b_drift': np.full(3, 5e-5), 'b_corr': np.array([np.inf, 100.0, 1.0]),
         'vrw': np.full(3, 0.03 / 60)}


def _k9_pair(eng, form, rg, ra, R, start, r0=2):
    """K9 of the call (end_err, proc) and K1's errors e [R, n, 6] of the same call."""
    gt, at = K9_FORMS[form]
    ge_, ae_ = dict(MID_G, **gt), dict(MID_A, **at)
    end, proc = eng.imu_err_stats(FS, R, eng.to_device(rg), eng.to_device(ra), ge_, ae_, SEED, run_offset=r0,
                                  stats_start=start)
    with np.errstate(invalid='ignore'):
        e = _k1(eng, R, len(rg), ge_, ae_, r0=r0, rg=rg, ra=ra) - np.concatenate([ra, rg], axis=1)[None]
    return end.cpu().numpy(), proc.cpu().numpy(), e


@pytest.mark.parametrize('form', list(K9_FORMS))
@pytest.mark.parametrize('n', [895, 896, 897, 2689])
def test_k9_tile_edges(eng, form, n):
    rng = np.random.default_rng(n)
    rg, ra = rng.standard_normal((n, 3)) * 0.3, rng.standard_normal((n, 3)) * 3.0 + [0.0, 0.0, -9.8]
    for start in sorted({s for s in (0, 3, 7, 896, n - 1) if s < n}):
        end, proc, e = _k9_pair(eng, form, rg, ra, 5, start)
        _same(end, e[:, -1], 'K9-%s end_err n %d' % (form, n))
        _check(proc, sx.per_run(e, start), e[:, start:], 1, DEPTH_K9, 'K9-%s n %d start %d' % (form, n, start), 'first')


@pytest.mark.parametrize('form', list(K9_FORMS))
def test_k9_end_err_where_the_drift_dominates(eng, form):
    """end_err bit for bit where a^q S is as large as the rest of the sample: ref = 0, no white noise, a strong
    drift on every channel, and the last sample at every position q = 0 .. 6 of its stretch (n = 890 .. 896), over
    64 runs.  A K9 that rounded a^q S before adding it would differ from K1's fused stage in some of them."""
    gt, at = K9_FORMS[form]
    gt, at = ({k: v for k, v in x.items() if k != 'b_std'} for x in (gt, at))    # b_run would dwarf the drift
    ge_ = dict(_zero('arw'), b_drift=np.full(3, 1e-2), b_corr=np.array([1.0, 0.5, 100.0]), **gt)
    ae_ = dict(_zero('vrw'), b_drift=np.full(3, 1e-1), b_corr=np.array([100.0, 2.0, 0.3]), **at)
    R = 64
    for n in range(890, 897):
        z = eng.to_device(np.zeros((n, 3)))
        end, _ = eng.imu_err_stats(FS, R, z, z, ge_, ae_, SEED, run_offset=R0)
        _same(end.cpu().numpy(), _k1(eng, R, n, ge_, ae_)[:, -1], 'K9-%s end_err n %d' % (form, n))


@pytest.mark.parametrize('form', list(K9_FORMS))
def test_k9_segmented_with_a_nan_in_the_third_segment(eng, form):
    """3 runs x 300 000 samples: a NaN ref_accel value inside the third segment.  Without run errors that column is
    NaN; with them all three accel columns are.  Every other column equals the clean launch bit for bit, the clean
    launch's statistics are K1's series', and end_err is K1's."""
    from gnss_ins_sim_b200 import _lib
    R, n, start = SEG_R, SEG_N, 100
    gt, at = K9_FORMS[form]
    plan = _lib.noise_plan(FS, R, n, dict(MID_G, **gt), dict(MID_A, **at))
    assert plan['nseg'] >= 3, plan
    rng = np.random.default_rng(6)
    rg, ra = rng.standard_normal((n, 3)) * 0.3, rng.standard_normal((n, 3)) * 3.0
    a2 = ra.copy()
    a2[2 * plan['seg_len'] + 5, 1] = np.nan
    end0, clean, e = _k9_pair(eng, form, rg, ra, R, start)
    _same(end0, e[:, -1], 'K9-%s segmented end_err' % form)
    _check(clean, sx.per_run(e, start), e[:, start:], 1, DEPTH_K9, 'K9-%s segmented' % form, 'first')
    end, proc, _ = _k9_pair(eng, form, rg, a2, R, start)
    _same(end, end0, 'K9-%s end_err with the NaN' % form)
    nan_cols = [0, 1, 2] if form != 'ex' else [1]
    assert np.isnan(proc[:, :, nan_cols]).all()
    others = np.ones(6, dtype=bool)
    others[nan_cols] = False
    _same(proc[:, :, others], clean[:, :, others], 'K9-%s segmented, other columns' % form)


@pytest.mark.parametrize('what', ['nan', 'inf'])
@pytest.mark.parametrize('form', list(K9_FORMS))
def test_k9_non_finite_reference_value(eng, form, what):
    """One NaN or inf in ref_accel column 1.  K1 with run errors: all three accel channels non-finite at that
    sample (NaN for a NaN; for an inf, +-inf or NaN, as terms_exact.run_err_sample makes them), the gyro
    unchanged; without, only that column.  K9 is the statistics of that series, the gyro columns and the other
    samples unchanged bit for bit."""
    n, R, start, row = 2000, 5, 300, 1234
    rng = np.random.default_rng(1)
    rg, ra = rng.standard_normal((n, 3)) * 0.3, rng.standard_normal((n, 3)) * 3.0
    a2 = ra.copy()
    a2[row, 1] = np.nan if what == 'nan' else np.inf
    _, clean, e0 = _k9_pair(eng, form, rg, ra, R, start)
    end, proc, e = _k9_pair(eng, form, rg, a2, R, start)
    bad = [0, 1, 2] if form != 'ex' else [1]
    assert not np.isfinite(e[:, row, bad]).any()
    if what == 'nan':
        assert np.isnan(e[:, row, bad]).all()
    good = np.ones(6, dtype=bool)
    good[bad] = False
    _same(e[:, row, good], e0[:, row, good], 'K1-%s row %d' % (form, row))
    keep = np.ones(n, dtype=bool)
    keep[row] = False
    _same(e[:, keep], e0[:, keep], 'K1-%s other samples' % form)
    if form != 'ex':
        # the three channels as the fma chain makes them, from the device's table
        gt, at = K9_FORMS[form]
        tab = eng.imu_run_errors(R, dict(MID_G, **gt), dict(MID_A, **at), SEED, run_offset=2).cpu().numpy()
        with np.errstate(invalid='ignore'):
            chain = np.stack([_fma_chain_plus(a2[row:row + 1], a2[row:row + 1], tab[r, 0])[0] for r in range(R)])
        assert np.isnan(e[:, row, 1]).all()             # the bad column itself: minus its own reference
        x, y = e[:, row, [0, 2]], chain[:, [0, 2]]
        assert np.array_equal(np.isnan(x), np.isnan(y)) and np.array_equal(x[np.isinf(y)], y[np.isinf(y)])
    _check(proc, sx.per_run(e, start), e[:, start:], 1, DEPTH_K9, 'K9-%s %s' % (form, what), 'first')
    _same(proc[:, :, 3:], clean[:, :, 3:], 'K9-%s gyro columns' % form)
    _same(end, e[:, -1], 'K9-%s end_err' % form)


# ---- the host twins ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('layout', [0, 2])
def test_host_twins_are_the_device_entry_points(eng, layout):
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    R, n = 4, 1800
    rg, ra = _ref(n)
    ge_, ae_ = dict(MID_G, **K9_FORMS['ex_rx'][0]), dict(MID_A, **K9_FORMS['ex_rx'][1])
    se_g, se_a, vib = _lib.sensor_err(ge_, 'arw'), _lib.sensor_err(ae_, 'vrw'), _lib.vib(None)
    tg, ta, xg, xa = _lib.noise_terms(ge_), _lib.noise_terms(ae_), _lib.run_err(ge_), _lib.run_err(ae_)
    shape = (R, n, 3) if layout == 0 else (R, 3, n)
    for name in ('ex', 'rx'):
        g, a = np.zeros(shape), np.zeros(shape)
        args = [FS, R, n, _lib.host_ptr(rg), _lib.host_ptr(ra), ctypes.byref(se_g), ctypes.byref(se_a), tg, ta,
                ctypes.byref(vib), ctypes.byref(vib), SEED, R0, layout, _lib.host_ptr(g), _lib.host_ptr(a), None]
        if name == 'ex':
            _lib.check(lib.b2ins_imu_noise_ex_f64_host(*args))
            want = eng.imu_noise(FS, R, eng.to_device(rg), eng.to_device(ra), dict(MID_G, **K9_FORMS['ex'][0]),
                                 dict(MID_A, **K9_FORMS['ex'][1]), SEED, run_offset=R0, layout=layout)
        else:
            _lib.check(lib.b2ins_imu_noise_rx_f64_host(*(args + [xg, xa])))
            want = eng.imu_noise(FS, R, eng.to_device(rg), eng.to_device(ra), ge_, ae_, SEED, run_offset=R0,
                                 layout=layout)
        _same(g, want[0].cpu().numpy(), 'imu_noise_%s_f64_host gyro' % name)
        _same(a, want[1].cpu().numpy(), 'imu_noise_%s_f64_host accel' % name)
    # K13 on K4's curves of those series, device and host
    gc = want[0] if layout == 2 else want[0].permute(0, 2, 1).contiguous()
    var, _ = eng.allan(FS, gc, n, R * 3)
    dev = eng.allan_fit(FS, n, var).cpu().numpy()
    v = var.cpu().numpy()
    host = np.zeros((R * 3, 6))
    _lib.check(lib.b2ins_allan_fit_f64_host(FS, n, R * 3, _lib.host_ptr(np.ascontiguousarray(v)), v.shape[-1], 1,
                                            _lib.host_ptr(host)))
    _same(host, dev, 'allan_fit_f64_host')
