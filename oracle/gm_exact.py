"""The exact Gauss-Markov bias drift of pathgen.bias_drift (pathgen.py:565-594), the reference of every drift
generator (K1 and K9, K12, the fused Allan front end).

For float64 a, b and drive normals z[0..n-1]:
    d_0 = 0,   d_{t+1} = a d_t + b z_t,   i.e.   d_t = sum_{k<t} a^(t-1-k) b z_k,
with b z_k the exact product of the two doubles (not rounded).  The recurrence runs in Python integers in
fixed point: every b z_k is an integer multiple of 2^-F with 64 bits to spare below the smallest of them, so
the products b z_k are exact and the one rounding per step of a d_t (half a unit of 2^-F) stays ~2^-64 below
the smallest drive over any series length used here.  Each d_t is then rounded once to float64.

The envelope the generators' bounds are written in,
    Psi_t = sum_{k<t} |a|^(t-1-k) (|b z_k| + |d_{k+1}|),
is returned as an upper bound: computed in float64 (two roundings of non-negative terms per step) and raised
by the relative error that can accumulate, (2 t + 4) u.

A white channel (tau = inf: a = b = 0, wd = b_drift) is d_t = fl(wd z_t), bit for bit; its Psi is 0."""
import math

import numpy as np
from scipy.signal import lfilter

U = 2.0 ** -53


def _mant_exp(x):
    """x = M 2^E with M an integer (numpy float64 array -> int64 mantissas, int64 exponents)."""
    m, e = np.frexp(np.asarray(x, dtype=np.float64))
    return (m * 2.0 ** 53).astype(np.int64), e.astype(np.int64) - 53


def _to_float(D, F):
    """D 2^-F rounded once to float64 (int / int is correctly rounded); +-inf past the float64 range."""
    try:
        return D / (1 << F) if F >= 0 else float(D << -F)
    except OverflowError:
        return math.copysign(math.inf, D)


def drift(a, b, z):
    """d [S, n] (float64, each correctly rounded) and Psi [S, n] (an upper bound) of S series.
    a, b: [S] float64 (or scalars); z: [S, n] (or [n]) float64 drive normals."""
    z = np.asarray(z, dtype=np.float64)
    one = z.ndim == 1
    z = np.atleast_2d(z)
    S, n = z.shape
    a = np.broadcast_to(np.asarray(a, dtype=np.float64), (S,))
    b = np.broadcast_to(np.asarray(b, dtype=np.float64), (S,))
    assert np.all(np.isfinite(a)) and np.all(np.isfinite(b)) and np.all(np.isfinite(z))
    Mz, Ez = _mant_exp(z)
    Mb, Eb = _mant_exp(b)
    live = (Mz != 0) & (Mb[:, None] != 0)
    lo = int((Eb[:, None] + Ez)[live].min()) if live.any() else 0
    F = 64 - lo                                     # the drives, in units of 2^-F, are integers times 2^64
    Ma, Ea = _mant_exp(a)
    d = np.zeros((S, n))
    for s in range(S):
        # b z_k / 2^-F = Mb Mz 2^(Eb + Ez + F): exact integers
        mb, sb = int(Mb[s]), int(Eb[s]) + F
        bz = [mb * m << (sb + e) if m and mb else 0 for m, e in zip(Mz[s].tolist(), Ez[s].tolist())]
        ma, k_sh = int(Ma[s]), -int(Ea[s])          # a D = ma D 2^-k_sh
        half = 1 << (k_sh - 1) if k_sh > 0 else 0
        out = [0.0] * n
        D = 0
        for t in range(1, n):
            P = ma * D
            D = (((P + half) >> k_sh) if k_sh > 0 else (P << -k_sh)) + bz[t - 1]   # round half up: <= 1/2
            out[t] = _to_float(D, F)
        d[s] = out
    # Psi: y_t = |a| y_{t-1} + x_t with x_t = |b z_{t-1}| + |d_t| (y_0 = 0), in float64, then raised
    x = np.zeros((S, n))
    x[:, 1:] = np.abs(b[:, None] * z[:, :-1]) + np.abs(d[:, 1:])
    psi = np.stack([lfilter([1.0], [1.0, -abs(a[s])], x[s]) for s in range(S)])
    psi *= 1.0 + (2.0 * np.arange(n) + 4.0) * U
    return (d[0], psi[0]) if one else (d, psi)


def channels(coef, z):
    """The exact drift of the six channels of every run: coef = _lib.noise_plan(...) (gm_a, gm_b, wd of
    accel x y z, gyro x y z), z [R, n, 6] the drive normals z0 of those channels (K1's z_dump[..., (0, 1, 2,
    6, 7, 8)]).  Returns d, Psi [R, n, 6]; white channels are fl(wd z), with Psi 0."""
    z = np.asarray(z, dtype=np.float64)
    R, n, _ = z.shape
    d = np.zeros((R, n, 6))
    psi = np.zeros((R, n, 6))
    for c in range(6):
        if coef['wd'][c] != 0.0 or (coef['gm_a'][c] == 0.0 and coef['gm_b'][c] == 0.0):
            d[:, :, c] = coef['wd'][c] * z[:, :, c]
            continue
        dc, pc = drift(np.full(R, coef['gm_a'][c]), np.full(R, coef['gm_b'][c]), z[:, :, c])
        d[:, :, c], psi[:, :, c] = dc, pc
    return d, psi


def z0_of_dump(zd):
    """K1's z_dump [R, n, 12] = (acc_gm[3], acc_w[3], gyr_gm[3], gyr_w[3]) -> the drives z0 [R, n, 6] of
    accel x y z, gyro x y z."""
    zd = np.asarray(zd, dtype=np.float64)
    return np.concatenate([zd[..., 0:3], zd[..., 6:9]], axis=-1)
