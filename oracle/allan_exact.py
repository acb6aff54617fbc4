"""The exact allan.allan_var (allan/allan.py:18-59), the reference of K4.

Every finite sample is an integer multiple of 2^E, E the exponent of the lowest set bit of any sample, so the
bin sums, the differences of adjacent sums and their squares are Python integers, and
    avar(m) = sum_b (B_{b+1} - B_b)^2 / (2 (nb - 1) m^2)
is rounded once, when that ratio of integers becomes a float64.  tau = m * (1 / fs), as allan.py:58 forms it;
the grid is oracle_np.allan_multipliers.

Non-finite samples follow IEEE arithmetic applied to the reference's own operations (np.mean over a bin, the
difference of adjacent means, its square, the sum over bins):
    a bin mean is NaN if the bin holds a NaN or both infinities, +-inf if it holds one sign of infinity;
    a difference is NaN for a NaN or for two infinities of the same sign, +-inf for one infinity;
    the sum is NaN if a term is NaN, otherwise +inf if a term is infinite.
Samples past nb * m do not count for that tau.
"""
import numpy as np

from oracle_np import allan_multipliers

_CHUNK = 2520 * 400      # level-0 samples per block: a multiple of every j = 1..9 and of 10


def _exponent(x):
    """E: every sample of x (finite) is an integer multiple of 2^E."""
    nz = x[x != 0.0]
    if nz.size == 0:
        return 0
    m, e = np.frexp(nz)
    return int((e.astype(np.int64) - 53).min())


def _ints(x, E):
    """x / 2^E as Python integers (exact)."""
    m, e = np.frexp(x)
    M = (m * 2.0 ** 53).astype(np.int64)
    sh = e.astype(np.int64) - 53 - E
    sh[M == 0] = 0
    return np.array([int(a) << int(b) for a, b in zip(M.tolist(), sh.tolist())], dtype=object)


def _ratio(num, den, E):
    """num * 2^(2E) / den rounded once to float64."""
    if num == 0:
        return 0.0
    if E < 0:
        den <<= -2 * E
    else:
        num <<= 2 * E
    try:
        return num / den          # int / int: correctly rounded
    except OverflowError:
        return np.inf


def _sum_sq_diff(bins):
    d = np.diff(bins)
    return int((d * d).sum()) if d.size else 0


def _finite_exact(x, mult):
    """sum_b D_b^2 per tau (integers, in units of 2^(2E)) and E, of a finite series."""
    n = len(x)
    E = _exponent(x)
    by_level = {}
    for i, m in enumerate(mult):
        k = len(str(m)) - 1
        by_level.setdefault(k, []).append((i, m // 10 ** k, n // m))
    acc = [0] * len(mult)
    # level 0 in blocks (a block starts a bin of every j), carrying each j's last bin sum across blocks
    prev = {}
    s = []
    for a in range(0, n, _CHUNK):
        b = min(n, a + _CHUNK)
        xi = _ints(x[a:b], E)
        for i, j, nb in by_level.get(0, []):
            hi = min(b, nb * j)
            if hi <= a:
                continue
            bins = xi[:hi - a].reshape(-1, j).sum(axis=1)
            if j in prev:
                bins = np.concatenate([[prev[j]], bins])
            acc[i] += _sum_sq_diff(bins)
            prev[j] = bins[-1]
        nd = (b - a) // 10
        if nd:
            s.append(xi[:10 * nd].reshape(nd, 10).sum(axis=1))
    s = np.concatenate(s) if s else np.zeros(0, dtype=object)
    k = 1
    while k in by_level:
        for i, j, nb in by_level[k]:
            acc[i] = _sum_sq_diff(s[:nb * j].reshape(nb, j).sum(axis=1))
        nd = len(s) // 10
        s = s[:10 * nd].reshape(nd, 10).sum(axis=1)
        k += 1
    return acc, E


def nonfinite_class(x, mult):
    """Per tau: 0 finite, 1 +inf, 2 NaN, by the rules of the module docstring."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    flags = [np.concatenate([[0], np.cumsum(f)]) for f in (np.isnan(x), x == np.inf, x == -np.inf)]
    out = np.zeros(len(mult), dtype=np.int64)
    for i, m in enumerate(mult):
        nb = n // m
        edges = np.arange(nb + 1) * m
        cnan, cpos, cneg = (f[edges[1:]] - f[edges[:-1]] for f in flags)
        mnan = (cnan > 0) | ((cpos > 0) & (cneg > 0))
        mpos = ~mnan & (cpos > 0)
        mneg = ~mnan & (cneg > 0)
        dnan = mnan[1:] | mnan[:-1] | (mpos[1:] & mpos[:-1]) | (mneg[1:] & mneg[:-1])
        dinf = mpos[1:] | mpos[:-1] | mneg[1:] | mneg[:-1]
        out[i] = 2 if dnan.any() else 1 if dinf.any() else 0
    return out


def allan_var(x, fs):
    """Returns (avar, tau) of allan.allan_var, avar exact to the last bit (one rounding)."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    mult = allan_multipliers(n, fs)
    if not mult:
        return np.array([]), np.array([])
    tau = np.asarray(mult, dtype=np.float64) * (1.0 / float(fs))
    fin = np.isfinite(x)
    acc, E = _finite_exact(np.where(fin, x, 0.0), mult)
    avar = np.array([_ratio(a, 2 * (n // m - 1) * m * m, E) for a, m in zip(acc, mult)])
    if not fin.all():
        cls = nonfinite_class(x, mult)
        avar[cls == 1] = np.inf
        avar[cls == 2] = np.nan
    return avar, tau
