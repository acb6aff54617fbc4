"""IEEE Std 952 terms of the IMU error model -- quantisation Q, rate random walk K, rate ramp R -- in NumPy: the
oracle of K1's and K9's _ex forms (b2ins_imu_noise_ex_f64, b2ins_imu_err_stats_ex_f64), on top of
oracle_np.imu_noise with the same draws.

Per axis c of sensor s (0 accel, 1 gyro), sample t, dt = 1/fs, with the terms of an imu_model dict ('q', 'rrw',
'rr'; absent = 0), added to the measurement K1 makes:
    rate random walk  w[0] = 0, w[t+1] = w[t] + K sqrt(dt) z0(t), z0 of the Box-Muller pair of draw 32 + 3 s + c
                      (the Gauss-Markov convention: state 0 at t = 0, the last draw unused)
    quantisation      e[t] = Q sqrt(12) (u[t] - 1/2), u[t] = uniform01 of the words (x1:x0) of draw 38 + 3 s + c;
                      rate error (e[t+1] - e[t]) / dt, so every sample has its two draws
    rate ramp         R (t dt), the same in every run

The exact expectations of the Allan variance (K4: non-overlapping, K4o: overlapping -- the same expectation) and of
the overlapping Hadamard variance at tau = m dt follow from writing each estimator's difference D = sum_t c_t y_t
(Allan: c = (-1, +1)/m over two adjacent clusters, AVAR = E D^2 / 2; Hadamard: (1, -2, 1)/m over three,
HVAR = E D^2 / 6) in terms of the drives:
    white N          y = N / sqrt(dt) z:              E D^2 = N^2 / dt sum c^2
    quantisation Q   D = 1/dt sum_s e_s (c_{s-1} - c_s):  E D^2 = Q^2 / dt^2 sum (jumps of c)^2
    random walk K    D = K sqrt(dt) sum_s z_s C_s, C_s = sum_{t>s} c_t:  E D^2 = K^2 dt sum C_s^2
    ramp R           D = R dt sum_t c_t t (deterministic)
giving
    Allan:    N^2/tau,  3 Q^2/tau^2,  K^2 dt (2 m^2 + 1) / (6 m) = K^2 tau / 3 + K^2 dt / (6 m),  R^2 tau^2 / 2
    Hadamard: N^2/tau, 10 Q^2/(3 tau^2), K^2 dt (m^2 + 1) / (6 m) = K^2 tau / 6 + K^2 dt / (6 m),  0
The terms are independent and zero-mean apart from the ramp, so the expectations add.  expect_by_sums restates the
sums over c for any m, which the tests hold the closed forms to.
"""
import math

import numpy as np

import oracle_np as onp

DRAW_RRW = 32       # +3*sensor+axis: rate-random-walk drive (z0)
DRAW_QUANT = 38     # +3*sensor+axis: quantisation uniform, words (x1:x0)
TERM_KEYS = ('q', 'rrw', 'rr')


def _three(err, key):
    return np.broadcast_to(np.asarray(err.get(key, 0.0), dtype=np.float64), (3,))


def uniform01(t, draw, run, seed):
    """uniform01 of common.cuh: ((x1:x0) >> 12) 2^-52 in [0, 1)."""
    run = np.asarray(run, dtype=np.uint64)
    seed = int(seed)
    x0, x1, _, _ = onp.philox4x32_10(t, draw, run & onp._MASK, run >> onp._S32,
                                     seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    return (((x1 << onp._S32) | x0) >> np.uint64(12)).astype(np.float64) * (2.0 ** -52)


def term_parts(fs, n, err, sensor, seed, run_ids):
    """(walk, quantisation rate error, ramp) of one sensor's triad, each [R, n, 3]."""
    dt = 1.0 / fs
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    r = run_ids[:, None, None]
    ax = np.arange(3, dtype=np.uint64)[None, None, :]
    t = np.arange(n, dtype=np.uint64)[None, :, None]
    K, Q, R = _three(err, 'rrw'), _three(err, 'q'), _three(err, 'rr')
    walk = np.zeros((len(run_ids), n, 3))
    if np.any(K != 0.0):
        z0, _ = onp.normal_pair(t, DRAW_RRW + 3 * sensor + ax, r, seed)
        walk[:, 1:] = np.cumsum((K * math.sqrt(dt)) * z0[:, :-1], axis=1)
    quant = np.zeros_like(walk)
    if np.any(Q != 0.0):
        u = uniform01(np.arange(n + 1, dtype=np.uint64)[None, :, None], DRAW_QUANT + 3 * sensor + ax, r, seed)
        e = (Q * math.sqrt(12.0)) * (u - 0.5)
        quant = (e[:, 1:] - e[:, :-1]) / dt
    ramp = np.broadcast_to(R * (np.arange(n, dtype=np.float64)[:, None] * dt), walk.shape)
    return walk, quant, ramp


def terms(fs, n, err, sensor, seed, run_ids):
    """The three terms of one sensor summed: walk + (quantisation + ramp), [R, n, 3]."""
    walk, quant, ramp = term_parts(fs, n, err, sensor, seed, run_ids)
    return walk + (quant + ramp)


def imu_noise(fs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_ids, vib_acc=None, vib_gyro=None):
    """oracle_np.imu_noise plus the terms: gyro, accel [R, n, 3]."""
    gyro, accel = onp.imu_noise(fs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_ids, vib_acc, vib_gyro)
    n = ref_gyro.shape[0]
    if any(k in gyro_err for k in TERM_KEYS):
        gyro = gyro + terms(fs, n, gyro_err, 1, seed, run_ids)
    if any(k in accel_err for k in TERM_KEYS):
        accel = accel + terms(fs, n, accel_err, 0, seed, run_ids)
    return gyro, accel


# ---- exact expectations at tau = m dt -------------------------------------------------------------------------
def allan_expect(m, dt, N=0.0, Q=0.0, K=0.0, R=0.0):
    """E of the Allan variance (K4 and K4o) of white N + quantisation Q + rate random walk K + ramp R."""
    m = np.asarray(m, dtype=np.float64)
    tau = m * dt
    return N * N / tau + 3.0 * Q * Q / (tau * tau) + K * K * dt * (2.0 * m * m + 1.0) / (6.0 * m) \
        + R * R * tau * tau / 2.0


def hadamard_expect(m, dt, N=0.0, Q=0.0, K=0.0, R=0.0):
    """E of the overlapping Hadamard variance; the ramp cancels exactly."""
    m = np.asarray(m, dtype=np.float64)
    tau = m * dt
    return N * N / tau + 10.0 * Q * Q / (3.0 * tau * tau) + K * K * dt * (m * m + 1.0) / (6.0 * m) + 0.0 * R


def _weights(m, kind):
    c = np.concatenate([np.full(m, -1.0), np.full(m, 1.0)]) / m if kind == 'allan' else \
        np.concatenate([np.full(m, 1.0), np.full(m, -2.0), np.full(m, 1.0)]) / m
    return c, (2.0 if kind == 'allan' else 6.0)


def expect_by_sums(m, dt, kind, N=0.0, Q=0.0, K=0.0, R=0.0):
    """The same expectations from the sums over the difference weights c (no closed form): the derivation's
    middle step, which the closed forms are held to."""
    c, norm = _weights(m, kind)
    jumps = np.diff(np.concatenate([[0.0], c, [0.0]]))
    tails = np.cumsum(c[::-1])[::-1][1:]       # C_s = sum_{t>s} c_t over the window (zero outside)
    ramp = R * dt * np.sum(c * np.arange(len(c)))
    e = N * N / dt * np.sum(c * c) + Q * Q / (dt * dt) * np.sum(jumps ** 2) + K * K * dt * np.sum(tails ** 2) \
        + ramp * ramp
    return e / norm



# ---- closure with the Allan noise identification (K13): what Allan(fit=True) reads back from this generator ---
# The law cases of allan_fit_np (100 Hz, 360 000 samples, the same white levels and terms), generated by THIS model:
# the walk starts at 0 and leaves its last draw unused, and quantisation is i.i.d. -- not allan_fit_np.law_series,
# whose walk takes its first draw and whose quantisation rounds a random-walk angle.  Each case: the output column,
# the true value (SI units, as imu_model stores 'q', 'rrw', 'rr'), the white level N of both sensors, and the
# ratio identified / true over the 720 gyro series of 240 runs of law_ratios (seed 1, runs 0..239): mean, standard
# deviation, and a per-series envelope from the smallest to the largest ratio, widened by 2 sd (and >= 0).  The fit
# may leave a term out (a ratio of 0: one ramp series in 720), so the ramp's envelope reaches 0.  The relative
# weighting biases the long-tau terms (K, R) low, as in allan_fit_np.LAWS.  The CPU tests regenerate them.
LAW_FS, LAW_N = 100.0, 360000
LAWS = {
    'rrw': dict(col=3, key='rrw', truth=3e-5, N=1e-4, mean=0.954, sd=0.0657, lo=0.478, hi=1.251),
    'rr': dict(col=4, key='rr', truth=1e-6, N=1e-3, mean=0.8863, sd=0.1091, lo=0.0, hi=1.352),
    'q': dict(col=0, key='q', truth=1e-5 / math.sqrt(12.0), N=1e-4, mean=1.0013, sd=0.0145, lo=0.912, hi=1.07),
}


def law_errs(kind):
    """The imu_model dicts (gyro, accel) of law case `kind`: white N, the term, nothing else."""
    c = LAWS[kind]
    base = {'b': np.zeros(3), 'b_drift': np.zeros(3), 'b_corr': np.full(3, np.inf), c['key']: np.full(3, c['truth'])}
    return dict(base, arw=np.full(3, c['N'])), dict(base, vrw=np.full(3, c['N']))


def law_gyro(kind, seed, run_ids, fs=LAW_FS, n=LAW_N):
    """The gyro series [R, n, 3] that imu_noise makes for law case `kind` on a zero reference, built from the gyro
    draws alone (b = 0, no drift: the measurement is the white noise plus the term, as imu_noise sums it)."""
    ge, _ = law_errs(kind)
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    t = np.arange(n, dtype=np.uint64)[None, :, None]
    ax = np.arange(3, dtype=np.uint64)[None, None, :]
    _, zw = onp.normal_pair(t, onp.PAIR_GYRO + ax, run_ids[:, None, None], seed)
    white = zw.copy()
    for c in range(3):
        white[:, :, c] = ge['arw'][c] / math.sqrt(1.0 / fs) * white[:, :, c]
    return white + terms(fs, n, ge, 1, seed, run_ids)


def law_ratios(kind, seed, run_ids, fs=LAW_FS, n=LAW_N):
    """Identified / true term of every gyro channel of the runs [R, 3]: allan_var then allan_fit_np.fit."""
    import allan_fit_np as af
    c = LAWS[kind]
    g = law_gyro(kind, seed, run_ids, fs, n)
    return np.array([[af.fit(onp.allan_var(g[r, :, a], fs)[0], n, fs)[c['col']] / c['truth'] for a in range(3)]
                     for r in range(g.shape[0])])


def law_check(kind, ratios):
    """Every ratio inside the case's envelope, and their mean within 5 standard errors of the oracle's (the errors
    of both ensembles)."""
    c = LAWS[kind]
    r = np.asarray(ratios, dtype=np.float64).reshape(-1)
    inside = bool(np.all((r >= c['lo']) & (r <= c['hi'])))
    se = c['sd'] * math.sqrt(1.0 / r.size + 1.0 / (3 * 240))
    return inside and abs(r.mean() - c['mean']) <= 5.0 * se, (r.min(), r.mean(), r.max())
