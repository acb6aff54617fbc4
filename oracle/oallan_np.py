"""Overlapping Allan variance (NIST SP 1065 eq. 10) on the reference's tau grid -- the oracle of K4o.

For one series x_0 .. x_{n-1} and each cluster size m of allan.allan_var's grid (oracle_np.allan_multipliers):
    S(k, m) = x_k + ... + x_{k+m-1},   M = n - 2m + 1,
    avar_o(m) = 1 / (2 m^2 M) * sum_{k<M} (S(k+m, m) - S(k, m))^2.

oallan_var        the prefix-sum form, C[i] = sum_{q<i} (x_q - x_0) in np.longdouble (the shift by x_0 does
                  not change the variance); O(n) per tau.  Series with a NaN give NaN at every tau; series
                  with +-inf take the definitional form.
oallan_var_brute  the definition itself: explicit window means, O(n m) per tau, IEEE arithmetic throughout
                  (so inf - inf is NaN exactly where a window pair produces it).
oallan_var_prefix64  the prefix-sum form in plain float64: loses the m = 1 differences of long or drifting
                  series, kept to show what the compensated prefix of K4o guards against.
"""
import numpy as np

from oracle_np import allan_multipliers


def _grid(n, fs):
    """The cluster sizes and tau = m * ts with ts = 1 / fs, as allan.py:58 forms it (K4's tau, bit for bit)."""
    mult = allan_multipliers(n, fs)
    return mult, np.asarray(mult, dtype=np.float64) * (1.0 / float(fs))


def _prefix_form(x, fs, dtype):
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    mult, tau = _grid(n, fs)
    if not mult:
        return np.array([]), np.array([])
    c = np.zeros(n + 1, dtype=dtype)
    c[1:] = np.cumsum((x - x[0]).astype(dtype))
    avar = np.zeros(len(mult))
    for i, m in enumerate(mult):
        M = n - 2 * m + 1
        d = c[2 * m:] - 2 * c[m:n + 1 - m] + c[:M]
        avar[i] = float(np.sum(d * d) / (2 * dtype(m) * m * M))
    return avar, tau


def oallan_var(x, fs):
    """Returns (avar, tau); the same tau as allan_var."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    if np.isnan(x).any():
        mult, tau = _grid(n, fs)
        return np.full(len(mult), np.nan), tau
    if not np.isfinite(x).all():
        return oallan_var_brute(x, fs)
    return _prefix_form(x, fs, np.longdouble)


def oallan_var_prefix64(x, fs):
    return _prefix_form(x, fs, np.float64)


def oallan_var_brute(x, fs):
    """The definition with explicit window means, in IEEE float64 arithmetic."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    mult, tau = _grid(n, fs)
    avar = np.zeros(len(mult))
    with np.errstate(invalid='ignore', over='ignore'):
        for i, m in enumerate(mult):
            M = n - 2 * m + 1
            w = np.lib.stride_tricks.sliding_window_view(x, m).sum(axis=1) / m   # mean of x[k:k+m]
            d = w[m:m + M] - w[:M]
            avar[i] = np.sum(d * d) / (2.0 * M)
    return avar, tau
