"""The exact IEEE Std 952 terms (quantisation, rate random walk, rate ramp) and run-to-run errors of K1's and K9's
_ex and _rx forms, built from the doubles the device uses: the reference of tests/test_gpu_terms_exact.py.

Coefficients, as digest_terms and digest_noise make them from the imu_model values Q, K, R (SI units):
    q = fl(Q fl(sqrt 12)),   k = fl(K fl(sqrt(dt))),   dt = fl(1 / fs)
Per axis of one sensor, sample t (noise952_np states the model):
    quantisation   e[t] = fl(q (u[t] - 1/2)), u[t] = uniform01 (an integer times 2^-52 in [0, 1), so u - 1/2 is
                   exact); the rate error fl(fl(e[t+1] - e[t]) / dt), bit for bit: the kernel rounds the same three
                   operations and nothing else
    ramp           fl(R fl(t dt)), bit for bit
    walk           w[0] = 0, w[t+1] = w[t] + k z0(t): gm_exact.drift(1, k, z0) with the device's own drive normals
                   (draw 32 + 3 s + c); its Psi, sum_{s<t} (|k z_s| + |w[s+1]|), is the envelope of the walk's error
    run errors     the stored sample of an IMU with only run errors set is
                   fl(ref_c + fma(S_c2, ref_2, fma(S_c1, ref_1, fma(S_c0, ref_0, b_c)))) (run_err_add), from the
                   device's own table (engine.imu_run_errors), through an exact fma

assemble() gives the exact sum of every component of a sample with everything set, and the bound of the kernel's
association order around it (its docstring derives the count)."""
import math
from fractions import Fraction

import numpy as np

import gm_exact as ge
import noise952_np as nz

U = 2.0 ** -53


def coefficients(fs, err):
    """(q [3], k [3], r [3], dt) of one sensor's imu_model dict, as the device holds them."""
    Q, K, R = (np.broadcast_to(np.asarray(err.get(key, 0.0), dtype=np.float64), (3,)) for key in ('q', 'rrw', 'rr'))
    dt = 1.0 / fs
    return Q * math.sqrt(12.0), K * math.sqrt(dt), R.copy(), dt


def fma(a, b, c):
    """a b + c rounded once (float64 scalars).  The exact value is a Fraction, whose conversion to float rounds
    correctly (int / int); an exact zero takes IEEE's sign from the float expression, which is exact then."""
    a, b, c = float(a), float(b), float(c)
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        return a * b + c                            # NaN and infinities propagate as the fused operation's do
    x = Fraction(a) * Fraction(b) + Fraction(c)
    if x == 0:
        return a * b + c
    try:
        return float(x)
    except OverflowError:
        return math.inf if x > 0 else -math.inf


fma_np = np.vectorize(fma, otypes=[np.float64])


def quant_rate(q, u, dt):
    """The quantisation rate error [..., n, 3] from the uniforms u [..., n + 1, 3] of samples 0 .. n."""
    e = q * (u - 0.5)
    return (e[..., 1:, :] - e[..., :-1, :]) / dt


def quant_uniforms(n, sensor, seed, run_ids):
    """uniform01 of draws 38 + 3 sensor + c at t = 0 .. n: [R, n + 1, 3] (integer arithmetic, exact)."""
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    t = np.arange(n + 1, dtype=np.uint64)[None, :, None]
    ax = np.arange(3, dtype=np.uint64)[None, None, :]
    return nz.uniform01(t, nz.DRAW_QUANT + 3 * sensor + ax, run_ids[:, None, None], seed)


def ramp(r, n, dt):
    """fl(R fl(t dt)) [n, 3]."""
    return r[None, :] * (np.arange(n, dtype=np.float64)[:, None] * dt)


def walk(k, z):
    """The exact walk of one sensor and its Psi, [R, n, 3] each: z [R, n, 3] the device's drive normals."""
    z = np.asarray(z, dtype=np.float64)
    R, n, _ = z.shape
    d, psi = np.zeros((R, n, 3)), np.zeros((R, n, 3))
    for c in range(3):
        if k[c] != 0.0:
            d[:, :, c], psi[:, :, c] = ge.drift(np.ones(R), np.full(R, k[c]), z[:, :, c])
    return d, psi


def run_err_sample(ref, tab):
    """The stored sample [R, n, 3] of an IMU whose only error is its run errors: ref [n, 3], tab [R, 3, 4] (row c =
    S[c][0..2], b_run[c]), in run_err_add's order, each fma rounded once."""
    ref = np.asarray(ref, dtype=np.float64)
    tab = np.asarray(tab, dtype=np.float64)
    d = np.broadcast_to(tab[:, None, :, 3], (tab.shape[0], ref.shape[0], 3))
    for j in range(3):
        d = fma_np(tab[:, None, :, j], ref[None, :, j:j + 1], d)
    with np.errstate(invalid='ignore'):
        return ref[None] + d


def run_err_exact(ref, tab):
    """b_run + S ref [R, n, 3] in exact arithmetic, rounded once, and sum |.| of its terms (its envelope)."""
    ref = np.asarray(ref, dtype=np.float64)
    tab = np.asarray(tab, dtype=np.float64)
    R, n = tab.shape[0], ref.shape[0]
    out = np.zeros((R, n, 3))
    env = np.abs(tab[:, None, :, 3]) + sum(np.abs(tab[:, None, :, j] * ref[None, :, j:j + 1]) for j in range(3))
    F = [[Fraction(float(v)) for v in row] for row in ref.tolist()]
    for r in range(R):
        for c in range(3):
            S = [Fraction(float(v)) for v in tab[r, c]]
            for t in range(n):
                out[r, t, c] = float(S[3] + S[0] * F[t][0] + S[1] * F[t][1] + S[2] * F[t][2])
    return out, env * (1.0 + 4 * U)


# The association order of one sample and channel in K1 (TERMS and RUNERR, no vibration), each step one rounding:
#   triad_sample   fl(ref + b), w z1 and its add, + r3 (the Gauss-Markov stretch partial), wd z0 and its add
#                  (each product fused into its add or not: 2 apiece)                                             6
#   terms_sample   qr + R (t dt) (fused or not: against the two exact components, 2), rk + that, m3 + that    4
#   run_err_add    the three fmas of delta and m3 + delta                                                      4
#   the stage      fma(a^q, S, .) (K1 by contraction, K9 written so) and + S_walk                              2
# and on the reference's side the drift and the walk, each rounded once, and the exact sum rounded once (3):
# N_ASM = 19.  Every value rounded is a partial sum of the components, whose magnitude is at most
#   M = |ref| + |b| + |w z1| + |wd z0| + |d| + 2 Psi_gm + |walk| + 2 Psi_walk + |quant| + |ramp|
#       + |b_run| + sum_j |S ref|
# (a stretch partial lies within Psi of its generator's zero, a^q S within |d| + Psi) to first order, and
# gamma_N = N u / (1 - N u) holds the rest.  The drift's and the walk's own scans add their bounds, C_gm u Psi_gm
# and C_walk u Psi_walk (each of which counts its stage adds once more: an upper count).
N_ASM = 19


def gamma(N):
    return N * U / (1.0 - N * U)


def assemble(ref, sens, z1, z0, gm, psi_gm, wlk, psi_walk, quant, rmp, tab, c_gm, c_walk):
    """The exact sum of every component of one sensor's samples [R, n, 3], rounded once, and its bound.
    ref [n, 3]; sens: dict of the digested triad b, w, wd [3] (the white products w z1, wd z0 are taken exactly);
    z1, z0 [R, n, 3] the device's normals; gm, psi_gm: gm_exact of the drift; wlk, psi_walk: walk(); quant, rmp:
    the exact term values; tab [R, 3, 4] the run-error table."""
    ref = np.asarray(ref, dtype=np.float64)
    R, n, _ = np.shape(gm)
    exact = np.zeros((R, n, 3))
    Fr = [[Fraction(float(v)) for v in row] for row in ref.tolist()]
    for c in range(3):
        b, w, wd = (Fraction(float(sens[k][c])) for k in ('b', 'w', 'wd'))
        for r in range(R):
            S = [Fraction(float(v)) for v in tab[r, c]]
            for t in range(n):
                x = (Fr[t][c] + b + w * Fraction(float(z1[r, t, c])) + wd * Fraction(float(z0[r, t, c])) +
                     Fraction(float(gm[r, t, c])) + Fraction(float(wlk[r, t, c])) + Fraction(float(quant[r, t, c])) +
                     Fraction(float(rmp[t, c])) + S[3] + S[0] * Fr[t][0] + S[1] * Fr[t][1] + S[2] * Fr[t][2])
                exact[r, t, c] = float(x)
    env = np.abs(tab[:, None, :, 3]) + sum(np.abs(tab[:, None, :, j] * ref[None, :, j:j + 1]) for j in range(3))
    M = (np.abs(ref)[None] + np.abs(sens['b']) + np.abs(sens['w'] * z1) + np.abs(sens['wd'] * z0) + np.abs(gm) +
         2 * psi_gm + np.abs(wlk) + 2 * psi_walk + np.abs(quant) + np.abs(rmp)[None] + env) * (1.0 + 4 * U)
    bound = gamma(N_ASM) * M + gamma(c_gm) * psi_gm + gamma(c_walk) * psi_walk
    return exact, bound
