"""The vibration series of a PSD table without the rounding of a float64 transform.

time_series_from_psd (oracle_np) takes the real part of the inverse DFT of the Hermitian spectrum built from
the L = N/2 + 1 bins A_k + j B_k.  That real part is the cosine synthesis

    x[m] = (1/N) [ A_0 + (-1)^m A_{L-1} + 2 sum_{k=1}^{L-2} (A_k cos(2 pi k m / N) - B_k sin(2 pi k m / N)) ]

which this module evaluates from the same bins (oracle_np.psd_bins): every angle reduced in integers,
r = k m mod N, and taken from a table of cos / sin(2 pi r / N) evaluated in np.longdouble, the products and
sums in np.longdouble as well.  Where np.longdouble is no wider than float64 the table and the products are
float64 and every sample is summed exactly by math.fsum.  Either way the result is good to a few 1e-16 of
the series maximum, far below what a float64 transform loses (~1e-15), so it can certify one."""
import math

import numpy as np

import oracle_np as onp

WIDE = np.finfo(np.longdouble).eps < np.finfo(np.float64).eps
_CHUNK = 1 << 20          # (m, k) terms per block


def cosine_synthesis(A, B, N):
    """x[0:N] (float64) of the bins A, B [L = N/2 + 1] of an even period N."""
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    L = N // 2 + 1
    assert N % 2 == 0 and A.shape == (L,) and B.shape == (L,), (N, A.shape, B.shape)
    dt = np.longdouble if WIDE else np.float64
    r = np.arange(N)
    if WIDE:
        two_pi = 2 * np.arccos(np.longdouble(-1))
        ang = two_pi * r.astype(dt) / dt(N)
    else:
        ang = 2.0 * np.pi * r / N
    cos_t, sin_t = np.cos(ang), np.sin(ang)
    k = np.arange(1, L - 1)
    a2, b2 = 2 * A[1:L - 1].astype(dt), 2 * B[1:L - 1].astype(dt)
    out = np.empty(N)
    rows = max(1, _CHUNK // max(1, k.size))
    for m0 in range(0, N, rows):
        m = np.arange(m0, min(N, m0 + rows))
        last = np.where(m % 2 == 0, A[L - 1], -A[L - 1])                # (-1)^m A_{L-1}, exact
        idx = (m[:, None] * k[None, :]) % N                              # k m mod N, in integers
        terms = a2 * cos_t[idx] - b2 * sin_t[idx]                        # [rows, L - 2]
        if WIDE:
            s = (terms.sum(axis=1) + dt(A[0])) + last.astype(dt)
            out[m0:m0 + m.size] = np.asarray(s / dt(N), dtype=np.float64)
        else:
            out[m0:m0 + m.size] = [math.fsum(list(t) + [A[0], e]) / N for t, e in zip(terms, last)]
    return out


def time_series_from_psd(sxx, freq, fs, n, phase_normals):
    """oracle_np.time_series_from_psd evaluated by cosine_synthesis: (ok, x[n]), tiled the same way."""
    bins = onp.psd_bins(sxx, freq, fs, n, phase_normals)
    if bins is None:
        return False, np.zeros((n,))
    N, xk = bins
    return True, onp.tile_period(cosine_synthesis(xk.real, xk.imag, N), n)
