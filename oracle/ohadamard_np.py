"""Overlapping Hadamard variance (NIST SP 1065) on the reference's tau grid -- the oracle of K4o's Hadamard form.

For one series x_0 .. x_{n-1} and each cluster size m of allan.allan_var's grid (oracle_np.allan_multipliers):
    S(k, m) = x_k + ... + x_{k+m-1},   H = n - 3m + 1,
    hvar(m) = 1 / (6 m^2 H) * sum_{k<H} (S(k+2m, m) - 2 S(k+m, m) + S(k, m))^2
            = 1 / (6 m^2 H) * sum_{k<H} (C[k+3m] - 3 C[k+2m] + 3 C[k+m] - C[k])^2,
with C[i] = sum_{q<i} (x_q - x_0).  A second difference of adjacent window sums: a linear drift of the samples
cancels exactly, white noise still gives sigma^2 / m.

ohadamard_var          the prefix form in np.longdouble; O(n) per tau.  Series with a NaN give NaN at every tau;
                       series with +-inf take the definitional form.
ohadamard_var_brute    the definition itself: explicit window means, IEEE arithmetic throughout.
ohadamard_var_prefix64 the prefix form in plain float64, kept to show what K4o's compensated prefix guards against.
ohadamard_var_fixed    the prefix form in exact integers, for series on one binary grid: once a drift has cancelled
                       in the term, the long-double prefix's own rounding shows at long tau.
"""
import numpy as np

from oallan_np import _grid


def _hadamard_prefix_form(x, fs, dtype):
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    mult, tau = _grid(n, fs)
    if not mult:
        return np.array([]), np.array([])
    c = np.zeros(n + 1, dtype=dtype)
    c[1:] = np.cumsum((x - x[0]).astype(dtype))
    hvar = np.zeros(len(mult))
    for i, m in enumerate(mult):
        H = n - 3 * m + 1
        d = c[3 * m:] - 3 * c[2 * m:n + 1 - m] + 3 * c[m:n + 1 - 2 * m] - c[:H]
        hvar[i] = float(np.sum(d * d) / (6 * dtype(m) * m * H))
    return hvar, tau


def ohadamard_var(x, fs):
    """Returns (hvar, tau); the same tau as allan_var.  NaN samples: NaN at every tau; +-inf: the definition."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    if np.isnan(x).any():
        mult, tau = _grid(n, fs)
        return np.full(len(mult), np.nan), tau
    if not np.isfinite(x).all():
        return ohadamard_var_brute(x, fs)
    return _hadamard_prefix_form(x, fs, np.longdouble)


def ohadamard_var_prefix64(x, fs):
    return _hadamard_prefix_form(x, fs, np.float64)


def ohadamard_var_fixed(x, fs):
    """The prefix form in exact integer arithmetic, for series whose shifted samples x - x_0 are exact in
    float64 and lie on one binary grid 2^-e within 2^50 of zero (e.g. every sample in one binade).  Every term
    below 2^64 grid units is exact; only the squares and their sum round (long double).  Where a linear drift
    cancels, the term is small beside the prefix and the long-double prefix's own rounding shows at long tau
    (4.5e-9 of hvar on x_i = 1e4 + 1e-3 i + 1e-3 noise, n = 1e6); this form has none.  Raises ValueError for
    other series."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    mult, tau = _grid(n, fs)
    d = x - x[0]
    nz = x[x != 0.0]
    e = int(-(np.frexp(nz)[1] - 53).min()) if nz.size else 0     # the finest ulp among the samples
    with np.errstate(over='ignore'):
        q = np.ldexp(d, e)
    if not (np.all(np.isfinite(x)) and np.all(q == np.rint(q)) and np.abs(q).max() < 2.0 ** 50):
        raise ValueError('the shifted series is not exact on one grid of 2^-%d within 2^50' % e)
    q = q.astype(np.int64)
    hi, lo = q >> 24, q & ((1 << 24) - 1)          # prefix sums of both stay below 2^63 for n < 2^24
    A = np.concatenate([[0], np.cumsum(hi)])
    B = np.concatenate([[0], np.cumsum(lo)])
    hvar = np.zeros(len(mult))
    for i, m in enumerate(mult):
        H = n - 3 * m + 1

        def third(c):
            return c[3 * m:] - 3 * c[2 * m:n + 1 - m] + 3 * c[m:n + 1 - 2 * m] - c[:H]
        # both third differences are exact below 2^53; their sum is one rounding, exact below 2^64
        t = np.ldexp(np.ldexp(third(A).astype(np.longdouble), 24) + third(B).astype(np.longdouble), -e)
        hvar[i] = float(np.sum(t * t) / (6 * np.longdouble(m) * m * H))
    return hvar, tau


def ohadamard_var_brute(x, fs):
    """The definition with explicit window means, in IEEE float64 arithmetic."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    mult, tau = _grid(n, fs)
    hvar = np.zeros(len(mult))
    with np.errstate(invalid='ignore', over='ignore'):
        for i, m in enumerate(mult):
            H = n - 3 * m + 1
            w = np.lib.stride_tricks.sliding_window_view(x, m).sum(axis=1) / m   # mean of x[k:k+m]
            d = w[2 * m:2 * m + H] - 2.0 * w[m:m + H] + w[:H]
            hvar[i] = np.sum(d * d) / (6.0 * H)
    return hvar, tau
