"""Every Gauss-Markov bias-drift generator held to the exact drift (oracle/gm_exact.py).

A drift-only IMU (ref = 0, b = 0, arw = vrw = 0) makes every stored sample the drift d_t alone, up to the
roundings of the generator: d[t+1] = a d[t] + b z0[t], d[0] = 0, with z0 the device's drive normals (K1's
z_dump; K12 and the fused Allan front end draw the same pairs).  The coefficients are the launch's own
(_lib.noise_plan).  A white channel (b_corr = inf) is fl(wd z0) bit for bit.

Sample bound.  |d^_t - d_t| <= C u Psi_t / (1 - C u), Psi_t = sum_{k<t} |a|^(t-1-k) (|b z_k| + |d_{k+1}|).
Every rounding of a generator is either of a zero-state partial response (|.| <= the |b z_k| terms it holds,
carried to t by |a|^(t-1-k)) or of a state d at some sample (a |d_{k+1}| term); a power a^m formed by products
of a has relative error <= (m - 1) u and weighs on the terms it multiplies.  C counts, for one term, the
roundings and power factors on its way to t, by the generator's association order:
  K1 / K9: b z (1), the thread's serial stretch (kNoisePer = 7 FMAs), the 5-level warp scan, <= 3 warp FMAs +
    the lane's FMA + S or the tile carry (5), a^q S and the add into the stage (2), and at most one tile's
    worth of power factors (kNoiseTile = 896: apow, the scan's products, pA or tA):  C = 916;
    with segments also pow(a, seg_len) (CUDA's pow: <= 2 ulp) and the carry chain's product and FMA (4), and
    the drives pass 1 drops, |a|^pass1_len < 1e-20 of Psi, once per segment end: C = 920 + 1e-20 / u nseg.
  K12: b z (1), log2 G scan FMAs, G - 1 power factors in the scan, a^j (j - 1 <= G - 1), the d FMA, a^G (G -
    1) and the carry FMA: C = 3 G + log2 G + 2, G the lane group (the attitude/velocity form: kAvRound = 8).
  Fused Allan front end: b z (1), kGenPer = 10 FMAs, 5 + 15 + 1 scan FMAs, S or the chunk carry (1), the
    output FMA (1) and one 5040-sample chunk's power factors: C = 5074.
No free tolerance: a generator that rounds a^q or a^j through float32, or drops drives older than 1e-10 of
the state, is outside these bounds by orders of magnitude.  The worst err / bound per generator is printed
at the end of the module.
"""
import math

import numpy as np
import pytest

import allan_exact as ae
import gm_exact as ge
import stats_exact as sx

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

U = 2.0 ** -53
FS = 100.0
DT = 1.0 / FS
C_K1 = 1 + 7 + 5 + 5 + 2 + 896
C_K1_SEG = C_K1 + 4
WORST = {}

# correlation times by the class of a = 1 - dt / tau
TAU = {'tau=100s': 100.0, 'near random walk': 1e7, 'tau=3dt': 3 * DT, 'a=0': DT, 'a=-1/3': 0.75 * DT,
       'a=-0.99': DT / 1.99, 'a=-1': DT / 2, 'white': np.inf}
# |a|^2680 = 1e-10: pass 1 would hold 2688 samples at a 1e-10 threshold, holds 5376 at 1e-20
TAU_2688 = DT / (1.0 - math.exp(math.log(1e-10) / 2680))


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    print('\nGauss-Markov drift: worst |generated - exact| / bound per generator: ' +
          ', '.join('%s %.3g' % kv for kv in sorted(WORST.items())))


def _errs(gyro_corr, accel_corr, gyro_drift=1.7e-5, accel_drift=2e-3):
    """Drift-only error models: b = 0, no white noise; b_drift = 0 where drift is 0."""
    def one(corr, drift, key):
        return {'b': np.zeros(3), 'b_drift': np.broadcast_to(np.asarray(drift, dtype=np.float64), (3,)).copy(),
                'b_corr': np.asarray(corr, dtype=np.float64).copy(), key: np.zeros(3)}
    return one(gyro_corr, gyro_drift, 'arw'), one(accel_corr, accel_drift, 'vrw')


def _k1(eng, R, n, ge_, ae_, seed, r0, layout=0):
    """K1 of a drift-only IMU: meas [R, n, 6] (accel x y z, gyro x y z) and z0 [R, n, 6]."""
    z = eng.to_device(np.zeros((n, 3)))
    gyro, accel, zd = eng.imu_noise(FS, R, z, z, ge_, ae_, seed, run_offset=r0, layout=layout, dump_z=True)
    if layout == eng.LAYOUT_TIME_MAJOR:
        gyro, accel = gyro.permute(2, 0, 1), accel.permute(2, 0, 1)
    elif layout == eng.LAYOUT_CHANNEL_MAJOR:
        gyro, accel = gyro.permute(0, 2, 1), accel.permute(0, 2, 1)
    meas = torch.cat([accel, gyro], dim=2).cpu().numpy()
    return meas, ge.z0_of_dump(zd.cpu().numpy())


def _check(got, d, psi, C, key, what, extra=None):
    """|got - d| <= C u Psi / (1 - C u) (+ extra) sample by sample; white channels (Psi = 0) bit for bit."""
    bound = C * U * psi / (1.0 - C * U)
    if extra is not None:
        bound = bound + extra
    err = np.abs(got - d)
    bad = ~(err <= bound)
    assert not bad.any(), '%s: %d samples out of bound, worst err %.3e / bound %.3e at %s' % (
        what, bad.sum(), err[bad].max(), bound[bad][np.argmax(err[bad])], np.argwhere(bad)[0].tolist())
    r = float(np.max(err / np.where(bound > 0, bound, np.inf), initial=0.0))
    WORST[key] = max(WORST.get(key, 0.0), r)
    return bound


def _exact(eng, R, n, ge_, ae_, z0):
    from gnss_ins_sim_b200 import _lib
    plan = _lib.noise_plan(FS, R, n, ge_, ae_)
    d, psi = ge.channels(plan, z0)
    return plan, d, psi


def _seg_extra(plan, psi):
    """The drives pass 1 drops: below 1e-20 of Psi at each segment end before t (|a| <= 1 wherever pass 1 is
    shorter than the segment)."""
    if plan['nseg'] == 1 or plan['pass1_len'] == plan['seg_len']:
        return None
    n = psi.shape[1]
    ends = np.minimum(np.arange(n)[None, :, None] // plan['seg_len'], plan['nseg'] - 1)
    return 1e-20 * ends * np.maximum.accumulate(psi, axis=1)


# ---- K1, one segment -------------------------------------------------------------------------------------
MIX_ALL = ([TAU['tau=100s'], TAU['a=-1/3'], TAU['a=-1']], [TAU['near random walk'], TAU['tau=3dt'], TAU['a=0']])
MIX_ALL2 = ([TAU['a=-0.99'], TAU['white'], TAU['tau=3dt']], [TAU['tau=100s'], TAU['white'], TAU['a=-1/3']])


@pytest.mark.parametrize('n', [1, 2, 7, 8, 895, 896, 897, 1793, 5041, 20011])
def test_k1_unsegmented_every_class(eng, n):
    R = 3 if n > 5000 else 5
    for mix, (g, a) in enumerate((MIX_ALL, MIX_ALL2)):
        ge_, ae_ = _errs(g, a, accel_drift=[0.0, 2e-3, 2e-3] if mix else 2e-3)   # one channel with b_drift = 0
        meas, z0 = _k1(eng, R, n, ge_, ae_, 11 + mix, 7)
        plan, d, psi = _exact(eng, R, n, ge_, ae_, z0)
        assert plan['nseg'] == 1
        _check(meas, d, psi, C_K1, 'K1', 'K1 n=%d mix %d' % (n, mix))
        if mix:
            assert np.all(meas[:, :, 0] == 0.0)                 # b_drift = 0 with tau finite: d = 0
            assert np.array_equal(meas[:, :, 4], d[:, :, 4])    # white: fl(wd z0)


@pytest.mark.parametrize('layout', [0, 1, 2])
def test_k1_ragged_run_counts_and_layouts(eng, layout):
    """Run counts that are not a multiple of anything, at a length inside the third tile, in every layout; the
    same runs bit for bit in every layout and in any launch that holds them."""
    n = 2 * 896 + 13
    ge_, ae_ = _errs(MIX_ALL[0], MIX_ALL[1])
    for R in (1, 3, 37):
        meas, z0 = _k1(eng, R, n, ge_, ae_, 5, 1000, layout)
        plan, d, psi = _exact(eng, R, n, ge_, ae_, z0)
        _check(meas, d, psi, C_K1, 'K1', 'K1 layout %d R=%d' % (layout, R))
        one, _ = _k1(eng, 1, n, ge_, ae_, 5, 1000 + R - 1, 0)
        assert np.array_equal(one[0], meas[-1])


# ---- K1 and K9, segmented ----------------------------------------------------------------------------------
SEG_MIXES = {
    # pass 1 shortened: every channel short, white or a <= 0.  a = -0.99 sets its length (5376 samples);
    # before the |a| rule it was ignored, and pass 1 held 896 samples (|a|^896 = 1.2e-4)
    'a=-0.99': ([TAU['a=-0.99'], TAU['a=-1/3'], TAU['white']], [TAU['a=0'], TAU['tau=3dt'], TAU['white']]),
    # shortened to the same 5376 samples by a = +0.991, whose drives 2688 samples old still weigh 1e-10
    'a=+0.991': ([TAU_2688, TAU['a=-1/3'], TAU['white']], [TAU['a=0'], TAU['tau=3dt'], TAU['white']]),
    # a = -1 never decays: the whole segment (896 samples before the |a| rule)
    'a=-1': ([TAU['a=-1'], TAU['a=-0.99'], TAU['white']], [TAU['a=-1/3'], TAU['a=0'], TAU['white']]),
    # a slow channel: the whole segment
    'slow': ([TAU['tau=100s'], TAU['near random walk'], TAU['a=-0.99']], [TAU['white'], TAU['a=-1'], 1.0]),
}
SEG_R, SEG_N = 3, 300001
_seg_cache = {}


def _segmented(eng, mix):
    if mix not in _seg_cache:
        ge_, ae_ = _errs(*SEG_MIXES[mix])
        meas, z0 = _k1(eng, SEG_R, SEG_N, ge_, ae_, 23, 4)
        plan, d, psi = _exact(eng, SEG_R, SEG_N, ge_, ae_, z0)
        _seg_cache[mix] = (ge_, ae_, meas, plan, d, psi)
    return _seg_cache[mix]


@pytest.mark.parametrize('mix', list(SEG_MIXES))
def test_k1_segmented(eng, mix):
    ge_, ae_, meas, plan, d, psi = _segmented(eng, mix)
    assert plan['nseg'] >= 3, plan
    _check(meas, d, psi, C_K1_SEG, 'K1 segmented', 'K1 segmented ' + mix, _seg_extra(plan, psi))
    if mix in ('a=-0.99', 'a=+0.991'):
        assert plan['pass1_len'] == 5376 < plan['seg_len']
    else:
        assert plan['pass1_len'] == plan['seg_len']


@pytest.mark.parametrize('mix', list(SEG_MIXES))
def test_k9_segmented(eng, mix):
    """K9 on the same IMUs: proc_stats from sample 0, inside a segment, on a segment boundary and inside the
    last segment against stats_exact of the exact drift.  Bound: the reducer's (chains of <= 64 additions,
    a Chan merge: stats_exact.assert_stats 'first') plus max|d^ - d| over the counted samples on each of max,
    mean and std; end_err within the sample bound of the last sample."""
    ge_, ae_, meas, plan, d, psi = _segmented(eng, mix)
    L = plan['seg_len']
    extra = _seg_extra(plan, psi)
    B = C_K1_SEG * U * psi / (1.0 - C_K1_SEG * U) + (0.0 if extra is None else extra)
    z = eng.to_device(np.zeros((SEG_N, 3)))
    for start in (0, L // 2 + 5, L, (plan['nseg'] - 1) * L + 77):
        end, proc = eng.imu_err_stats(FS, SEG_R, z, z, ge_, ae_, 23, run_offset=4, stats_start=start)
        end, proc = end.cpu().numpy(), proc.cpu().numpy()
        assert np.all(np.abs(end - d[:, -1]) <= B[:, -1]), (mix, start)
        ex = sx.per_run(d, start)
        slack = B[:, start:].max(1)
        sx.assert_stats(proc, ex, 64 * sx.EPS * np.abs(d[:, start:]).max(1) * (1 + 1e-9), 64 * sx.EPS,
                        'K9 %s start %d' % (mix, start), 'first', max_exact=False, abs_slack=slack)
        with np.errstate(invalid='ignore', divide='ignore'):
            r = np.abs(proc - ex) / (np.abs(ex) * 64 * sx.EPS + slack[:, None, :])
        WORST['K9'] = max(WORST.get('K9', 0.0), float(np.nanmax(r)))


# ---- K12 -------------------------------------------------------------------------------------------------
def _c_k12(lanes, shape):
    G = lanes
    if shape == '' or (shape != '0' and shape.split(',')[1] != '1'):
        G = max(G, 8)                      # the attitude/velocity form (the default for some) scans rounds of 8
    return 3 * G + int(math.log2(G)) + 2


def _k12(eng, rf, R, n, lanes, ge_, ae_, seed, r0, shape, monkeypatch):
    from conftest import load_golden
    g = load_golden('philox_90deg_mid_rf%d.npz' % rf)
    nav = np.concatenate([g['ref_att'], g['ref_pos'], g['ref_vel']], axis=1)
    reps = -(-n // nav.shape[0])
    nav = np.concatenate([nav] * reps)[:n]
    zero = np.zeros((n, 3))
    dev = [eng.to_device(a) for a in (zero, zero, nav, g['ini'][None])]
    if shape:
        monkeypatch.setenv('B2INS_MC_SHAPE', shape)
    else:
        monkeypatch.delenv('B2INS_MC_SHAPE', raising=False)
    try:
        cfg = eng.make_mc_config(rf, FS, n, R, seed, ge_, ae_, 1, 9, lanes_per_run=lanes, dump_runs=R,
                                 run_offset=r0)
        res = eng.mc_free_integration(cfg, *dev, dump_imu=True)
    finally:
        monkeypatch.delenv('B2INS_MC_SHAPE', raising=False)
    return np.concatenate([res.accel.cpu().numpy(), res.gyro.cpu().numpy()], axis=2)


@pytest.mark.parametrize('rf', [1, 0])
def test_k12_every_launch_shape(eng, rf, monkeypatch):
    from test_gpu_r02 import SHAPES
    n, R = 1000, 8
    ge_, ae_ = _errs(MIX_ALL[0], MIX_ALL[1])
    _, z0 = _k1(eng, R, n, ge_, ae_, 31, 3)
    _, d, psi = _exact(eng, R, n, ge_, ae_, z0)
    for lanes, shape in SHAPES:
        try:
            got = _k12(eng, rf, R, n, lanes, ge_, ae_, 31, 3, shape, monkeypatch)
        except ValueError as e:
            assert 'no specialised kernel' in str(e), (lanes, shape, e)
            continue
        _check(got, d, psi, _c_k12(lanes, shape), 'K12', 'K12 rf %d lanes %d shape %s' % (rf, lanes, shape))


@pytest.mark.parametrize('rf', [1, 0])
def test_k12_ragged_runs_and_lengths(eng, rf, monkeypatch):
    """test_gpu_r02's ragged run counts, lane groups and lengths, plus a length over many 128-sample tiles."""
    ge_, ae_ = _errs(MIX_ALL2[0], MIX_ALL2[1])
    cases = [(1, 4, ''), (9, 4, ''), (33, 1, ''), (5, 8, ''), (3, 16, ''), (37, 2, ''),
             (9, 4, '6,1,0'), (5, 8, '6,1,0'), (9, 4, '6,1,1')]
    if rf == 1:
        cases += [(9, 4, '6,2,0'), (5, 8, '6,2,0'), (1, 4, '6,2,0')]
    for n in (1, 2, 4, 5, 7, 9, 129, 131, 777, 128 * 23 + 61):
        _, z0 = _k1(eng, 37, n, ge_, ae_, 99, 1000)
        _, d, psi = _exact(eng, 37, n, ge_, ae_, z0)
        for R, lanes, spec in cases:
            for shape in (spec, '0'):
                got = _k12(eng, rf, R, n, lanes, ge_, ae_, 99, 1000, shape, monkeypatch)
                _check(got, d[:R], psi[:R], _c_k12(lanes, shape or ''), 'K12',
                       'K12 rf %d n %d R %d lanes %d shape %r' % (rf, n, R, lanes, shape))


# ---- the fused Allan front end ---------------------------------------------------------------------------
C_ALLAN = 1 + 10 + 5 + 15 + 1 + 1 + 1 + 5040


def _allan_bound(d, B, fs, exact):
    """k4_bound of the series plus the sample bound B carried through the estimator: each difference of
    adjacent bin sums moves by at most beta = the B of both bins, its square by beta (2 |D| + beta)."""
    from test_gpu_allan_edges import k4_bound
    import oracle_np as onp
    n = len(d)
    out = k4_bound(d, fs, exact)
    for i, m in enumerate(onp.allan_multipliers(n, fs)):
        nb = n // m
        bs = d[:nb * m].reshape(nb, m).sum(1)
        Bs = B[:nb * m].reshape(nb, m).sum(1)
        D, beta = np.abs(np.diff(bs)), Bs[1:] + Bs[:-1]
        out[i] += (0.5 / ((nb - 1) * float(m) * m) * np.sum(beta * (2 * D + beta)) * (1 + 1e-6)
                   + 2 * U * exact[i])
    return out


@pytest.mark.parametrize('n', [3 * 5040 + 17, 10081])
def test_fused_allan_front_end(eng, n):
    """allan_mc: several 5040-sample chunks per series, more series than CTAs (every CTA walks several);
    avar of every series against allan_exact of the exact drift."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    R = sms // 6 + 3
    assert 6 * R > sms
    ge_, ae_ = _errs([TAU['tau=100s'], TAU['a=-1/3'], TAU['a=-0.99']],
                     [TAU['near random walk'], TAU['tau=3dt'], TAU['a=-1']])
    zero = eng.to_device(np.zeros((n, 3)))
    avar, tau = eng.allan_mc(FS, R, zero, zero, ge_, ae_, 17, run_offset=9)
    avar = avar.cpu().numpy()
    _, z0 = _k1(eng, R, n, ge_, ae_, 17, 9)
    _, d, psi = _exact(eng, R, n, ge_, ae_, z0)
    B = C_ALLAN * U * psi / (1.0 - C_ALLAN * U)
    for r in range(R):
        for c in range(6):
            ex, et = ae.allan_var(d[r, :, c], FS)
            assert np.array_equal(tau.cpu().numpy(), et)
            bound = _allan_bound(d[r, :, c], B[r, :, c], FS, ex)
            err = np.abs(avar[r, c] - ex)
            assert np.all(err <= bound), ('allan run %d ch %d' % (r, c), np.max(err / bound))
            WORST['allan_mc'] = max(WORST.get('allan_mc', 0.0), float(np.max(err / bound)))


# ---- Sim --------------------------------------------------------------------------------------------------
def test_sim_dict_imu_with_correlation_time_below_dt(eng):
    """A dict IMU with gyro_b_corr below dt (a = -1, -0.99 and -1/3) through Sim.get_data(['gyro']) for two
    runs of 300 001 samples: the segmented K1 path, against the exact drift."""
    from gnss_ins_sim_b200 import imu_model, _lib
    from gnss_ins_sim_b200.sim import Sim
    n, R = SEG_N, 2
    acc = {'gyro_b': np.zeros(3), 'gyro_arw': np.zeros(3), 'gyro_b_stability': np.array([3.5, 2.0, 5.0]),
           'gyro_b_corr': np.array([DT / 2, DT / 1.99, 0.75 * DT]),
           'accel_b': np.zeros(3), 'accel_vrw': np.zeros(3), 'accel_b_stability': np.full(3, 5e-5)}
    imu = imu_model.IMU(accuracy=acc, axis=6, gps=False)
    z = np.zeros((n, 3))
    traj = {'ref_pos': z, 'ref_vel': z, 'ref_att': z, 'ref_accel': z, 'ref_gyro': z}
    sim = Sim([FS, 0.0, 0.0], traj, ref_frame=1, imu=imu, seed=41)
    sim.run(R)
    gyro = sim.get_data(['gyro'])[0]
    plan = _lib.noise_plan(FS, R, n, imu.gyro_err, imu.accel_err)
    assert plan['nseg'] >= 3 and plan['pass1_len'] == plan['seg_len'] and plan['gm_a'][3] == -1.0
    _, z0 = _k1(eng, R, n, imu.gyro_err, imu.accel_err, 41, 0)
    d, psi = ge.channels(plan, z0)
    for r in range(R):
        _check(gyro[r][None], d[r:r + 1, :, 3:], psi[r:r + 1, :, 3:], C_K1_SEG, 'K1 segmented', 'Sim run %d' % r)


# ---- |a| > 1 --------------------------------------------------------------------------------------------
def test_growing_drift_while_the_reference_is_finite(eng):
    """tau < dt / 2 gives |a| > 1 (a = -3 at tau = dt / 4): the drift grows as 3^t and the reference stays
    finite up to ~640 samples.  Held to the bound at 600 samples on K1 and K12."""
    n, R = 600, 2
    ge_, ae_ = _errs([DT / 4, 0.4 * DT, TAU['white']], [TAU['white'], DT / 4, TAU['a=-1']])
    meas, z0 = _k1(eng, R, n, ge_, ae_, 3, 0)
    _, d, psi = _exact(eng, R, n, ge_, ae_, z0)
    assert np.all(np.isfinite(d)) and np.all(np.isfinite(psi)) and np.abs(d).max() > 1e200
    _check(meas, d, psi, C_K1, 'K1', 'K1 |a| > 1')
