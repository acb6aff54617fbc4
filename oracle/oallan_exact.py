"""The exact overlapping Allan variance and overlapping Hadamard variance, the reference of K4o.

For one series x_0 .. x_{n-1} and each cluster size m of K4's grid (oallan_np._grid, tau bit for bit):
    avar_o(m) = 1 / (2 m^2 M) * sum_{k<M} t_k^2,   t_k = S(k+m, m) - S(k, m),                     M = n - 2m + 1,
    hvar(m)   = 1 / (6 m^2 H) * sum_{k<H} t_k^2,   t_k = S(k+2m, m) - 2 S(k+m, m) + S(k, m),       H = n - 3m + 1,
with S(k, m) = x_k + ... + x_{k+m-1}.  Every finite sample is an integer multiple of 2^E, E the exponent of the
lowest set bit of any sample (allan_exact._exponent), so the prefix P[i] = sum_{q<i} x_q / 2^E, every term
t_k = P[k+2m] - 2 P[k+m] + P[k] (Allan) or P[k+3m] - 3 P[k+2m] + 3 P[k+m] - P[k] (Hadamard), and sum t_k^2 are
integers.  The variance is rounded once, when that integer over the exact integer 2 m^2 M (6 m^2 H) becomes a
float64 (allan_exact._ratio); a ratio above DBL_MAX is +inf.  No x - x_0 is ever formed in floating point.

Two paths compute the same integers:
  limbs  each sample split into signed int64 limbs of 2^20 (vectorised, O(n) NumPy work per limb and tau).  A term
         is normalised to balanced digits in [-2^19, 2^19), and sum t^2 is accumulated per digit pair in int64.
         Taken when n < 2^26 and the samples span at most MAX_LIMBS * 20 bits of 2^E (every finite series of one
         sensor, to well beyond 14.4 M samples).
  ints   Python integers (object arrays), for any other series: samples spanning more than 240 bits (e.g. 1e-300
         beside 1e300) or longer series.  About 0.1 s per tau at n = 2e5.

Non-finite samples (the rule of K4o's header comment, which is what the definitional sum gives in IEEE
arithmetic whatever the order of its additions), from per-tau prefix counts of NaN, +inf and -inf:
    a NaN sample makes every tau NaN;
    otherwise, with a +-inf sample, a tau is NaN if one of its terms is NaN, else +inf (every sample lies in a
    window of some term);
    an Allan term is NaN when one window holds both infinities or both windows hold the same one;
    a Hadamard term +S2 - 2 S1 + S0 is NaN when its signed contributions hold both infinities.

exact() also returns, per tau, max |t| and sum t^2 as floats, and hands the float64 terms (each within a few ulp
of the exact t_k) to a callback: what a bound on an estimator's rounding needs.  k4o_bound() is that bound for K4o,
derived step by step in tests/test_gpu_oallan_edges.py.
"""
import numpy as np

from allan_exact import _exponent, _ints, _ratio
from oallan_np import _grid

B = 20                       # bits per limb
MASK = (1 << B) - 1
HALF = 1 << (B - 1)
MAX_LIMBS = 12
MAX_N_LIMBS = 1 << 26        # prefix limbs stay below 2^46, a Hadamard term's below 2^49


def _diff(P, m, had):
    """The term of every offset from a prefix (limb array [..., n + 1] or object array)."""
    n = P.shape[-1] - 1
    if had:
        H = n - 3 * m + 1
        return P[..., 3 * m:] - 3 * P[..., 2 * m:2 * m + H] + 3 * P[..., m:m + H] - P[..., :H]
    M = n - 2 * m + 1
    return P[..., 2 * m:] - 2 * P[..., m:m + M] + P[..., :M]


def _limbs(x, E):
    """x / 2^E as signed int64 limbs [L, n] of 2^B: sum_l limb[l] * 2^(B l) is the integer, exactly."""
    m, e = np.frexp(x)
    M = (m * 2.0 ** 53).astype(np.int64)
    sh = e.astype(np.int64) - 53 - E
    sh[M == 0] = 0
    a = np.abs(M)
    L = int((sh + 53).max()) // B + 1 if len(x) else 1
    out = np.empty((L, len(x)), dtype=np.int64)
    for l in range(L):
        lo = B * l - sh                      # the bit of |M| that lands on bit 0 of limb l
        up = (a >> np.clip(lo, 0, 63)) & MASK
        left = np.clip(-lo, 0, B)
        down = (a & (MASK >> left)) << left
        v = np.where(lo >= 0, up, down)
        out[l] = np.where(M < 0, -v, v)
    return out


def _limb_count(x, E):
    m, e = np.frexp(x)
    return (int((e.astype(np.int64) - E).max()) // B + 1) if len(x) else 1


def _digits(T):
    """Limb terms [L, K] -> balanced digits [L', K] in [-2^(B-1), 2^(B-1)), the same integers."""
    L, K = T.shape
    out = []
    carry = np.zeros(K, dtype=np.int64)
    l = 0
    while l < L or carry.any():
        v = (T[l] if l < L else 0) + carry
        d = ((v + HALF) & MASK) - HALF
        carry = (v - d) >> B
        out.append(d)
        l += 1
    while len(out) > 1 and not out[-1].any():
        out.pop()
    return np.array(out)


def _sum_sq_limbs(d):
    """sum_k (sum_l d[l, k] 2^(B l))^2 as a Python integer; |d| < 2^(B-1), so each pair product is below 2^38."""
    L = d.shape[0]
    tot = 0
    for s in range(2 * L - 1):
        g = np.zeros(d.shape[1], dtype=np.int64)
        for l in range(max(0, s - L + 1), min(L, s + 1)):
            if 2 * l < s:
                g += 2 * d[l] * d[s - l]
            elif 2 * l == s:
                g += d[l] * d[l]
        # g < 2^(38 + 1 + log2 L): split it so that the sums over up to 2^26 terms stay in int64
        tot += ((int((g >> 24).sum()) << 24) + int((g & 0xFFFFFF).sum())) << (B * s)
    return tot


def _digits_float(d, E):
    """The terms in float64 (each digit exact; summed from the top, within a few ulp of t)."""
    f = np.zeros(d.shape[1])
    with np.errstate(over='ignore'):
        for l in range(d.shape[0] - 1, -1, -1):
            f += np.ldexp(d[l].astype(np.float64), B * l + E)
    return f


def _int_float(v, E):
    """Python integer v times 2^E as a float64 (inf past DBL_MAX), to a few ulp."""
    v = int(v)
    s = max(v.bit_length() - 60, 0)
    with np.errstate(over='ignore'):
        return float(np.ldexp(float(v >> s if v >= 0 else -((-v) >> s)), s + E))


def _path(n, L):
    return 'limbs' if n < MAX_N_LIMBS and L <= MAX_LIMBS else 'ints'


def classes(x, mult, hadamard=False):
    """Per tau: 0 finite, 1 +inf, 2 NaN, by the rule of the module docstring (O(n) per tau)."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    out = np.zeros(len(mult), dtype=np.int64)
    if np.isnan(x).any():
        out[:] = 2
        return out
    if np.isfinite(x).all():
        return out
    cp, cm = (np.concatenate([[0], np.cumsum(f)]) for f in (x == np.inf, x == -np.inf))
    for i, m in enumerate(mult):
        K = n - (3 if hadamard else 2) * m + 1
        k = np.arange(K)
        win = [(cp[k + (w + 1) * m] - cp[k + w * m] > 0, cm[k + (w + 1) * m] - cm[k + w * m] > 0)
               for w in range(3 if hadamard else 2)]
        if hadamard:
            (p0, n0), (p1, n1), (p2, n2) = win
            nan = (p0 | n1 | p2) & (n0 | p1 | n2)
        else:
            (pa, na), (pb, nb) = win
            nan = (pa & na) | (pb & nb) | (pa & pb) | (na & nb)
        out[i] = 2 if nan.any() else 1
    return out


def exact(x, fs, hadamard=False, mult=None, per_tau=None, path=None):
    """Returns (var, tau, info): the exact variance per tau (one rounding), tau = m * (1 / fs), and info with
    'cls' (0 finite, 1 +inf, 2 NaN), 'tmax' (max |t_k|), 'st2' (sum t_k^2, a float), 'path', and 'per_tau': the
    values of per_tau(i, m, t) for the float64 terms t of every tau (of the finite samples), if given.  mult: a
    subset of the grid (default all of it); path: 'limbs' or 'ints' to force one (limbs raises ValueError where it
    does not apply)."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    grid, _ = _grid(n, fs)
    mult = grid if mult is None else [int(m) for m in mult]
    assert set(mult) <= set(grid), mult
    tau = np.asarray(mult, dtype=np.float64) * (1.0 / float(fs))
    info = {'cls': classes(x, mult, hadamard), 'tmax': np.zeros(len(mult)), 'st2': np.zeros(len(mult)),
            'per_tau': []}
    var = np.zeros(len(mult))
    if not mult:
        info['path'] = None
        return var, tau, info
    xf = np.where(np.isfinite(x), x, 0.0)
    E = _exponent(xf)
    auto = _path(n, _limb_count(xf, E))
    path = path or auto
    if path == 'limbs' and auto != 'limbs':
        raise ValueError('the limb path needs n < 2^26 and at most %d limbs of 2^%d' % (MAX_LIMBS, B))
    info['path'] = path
    P = None
    if path == 'limbs':
        q = _limbs(xf, E)
        P = np.zeros((q.shape[0], n + 1), dtype=np.int64)
        np.cumsum(q, axis=1, out=P[:, 1:])
    else:
        P = np.concatenate([np.array([0], dtype=object), np.cumsum(_ints(xf, E))])
    den_k = 6 if hadamard else 2
    for i, m in enumerate(mult):
        K = n - (3 if hadamard else 2) * m + 1
        if path == 'limbs':
            d = _digits(_diff(P, m, hadamard))
            s2 = _sum_sq_limbs(d)
            tf = _digits_float(d, E)
        else:
            T = _diff(P, m, hadamard)
            s2 = int((T * T).sum())
            tf = np.array([_int_float(v, E) for v in T])
        var[i] = _ratio(s2, den_k * m * m * K, E)
        info['tmax'][i] = np.abs(tf).max()
        info['st2'][i] = _int_float(s2, 2 * E)
        if per_tau is not None:
            info['per_tau'].append(per_tau(i, m, tf))
    cls = info['cls']
    var[cls == 1] = np.inf
    var[cls == 2] = np.nan
    return var, tau, info


def oallan_var(x, fs, mult=None):
    """(avar_o, tau), exact to the last bit."""
    v, t, _ = exact(x, fs, False, mult)
    return v, t


def ohadamard_var(x, fs, mult=None):
    """(hvar, tau), exact to the last bit."""
    v, t, _ = exact(x, fs, True, mult)
    return v, t


# ---------------------------------------------------------------------------------------------------------------
# the bound of K4o's rounding (tests/test_gpu_oallan_edges.py derives it)
# ---------------------------------------------------------------------------------------------------------------
U = 2.0 ** -53
SCAN_TILE, SQ_TILE = 2304, 2048


def _gamma(p):
    return p * U / (1.0 - p * U)


def _two_sum_err(a, b):
    s = a + b
    bb = s - a
    return (a - (s - bb)) + (b - bb)


def _sterbenz(a, b):
    """a - b is exact in float64 (with a margin for a and b being the rounded hi parts)."""
    aa, ab = np.abs(a), np.abs(b)
    return (np.sign(a) == np.sign(b)) & (np.maximum(aa, ab) <= 2.0 * (1.0 - 1e-9) * np.minimum(aa, ab))


class _K4oBound:
    """Per-sample quantities of one finite series; __call__(i, m, t) is the bound of one tau."""

    def __init__(self, x, hadamard):
        x = np.asarray(x, dtype=np.float64)
        n = len(x)
        self.n, self.had = n, hadamard
        with np.errstate(over='ignore', invalid='ignore'):
            y = x - x[0]                                   # pass 1 and pass 3 round here
            dl = np.abs(_two_sum_err(x, -x[0]))            # the rounding of each x - x_0, exactly
        self.delta = np.concatenate([[0.0], np.cumsum(dl.astype(np.longdouble))])
        c = np.concatenate([[0.0], np.cumsum(x.astype(np.longdouble) - np.longdouble(x[0]))])
        self.c = c                                         # C within ~1e-19 |C|: magnitudes only
        a = np.concatenate([[0.0], np.cumsum(np.abs(y).astype(np.longdouble))]).astype(np.float64)
        tile = np.concatenate([[0], (np.arange(1, n + 1) - 1) // SCAN_TILE])
        # the double-double prefix: every element passes <= tile + 20 adds on its way to C[i], each add
        # erring by <= 8 u^2 (|a| + |b|)
        self.eps = 8.0 * U * U * a * (tile + 20) * (1.0 + 1e-6)
        self.sq_tiles = -(-n // SQ_TILE)

    def __call__(self, i, m, t):
        n, c, eps, dlt = self.n, self.c, self.eps, self.delta
        w = 3 if self.had else 2
        K = n - w * m + 1
        k = np.arange(K)
        idx = [k + j * m for j in range(w + 1)]
        C = [np.abs(c[q]).astype(np.float64) for q in idx]
        win = [(dlt[idx[j + 1]] - dlt[idx[j]]).astype(np.float64) for j in range(w)]
        at = np.abs(t)
        if self.had:
            S = [c[idx[j + 1]] - c[idx[j]] for j in range(3)]
            F2, F1 = (S[2] - S[1]).astype(np.float64), (S[1] - S[0]).astype(np.float64)
            S = [s.astype(np.float64) for s in S]
            lam = U * (np.abs(S[0]) + 2 * np.abs(S[1]) + np.abs(S[2])) + U * (C[0] + 3 * C[1] + 3 * C[2] + C[3])
            e = (2 * U * at + U * np.where(_sterbenz(S[2], S[1]), 0.0, np.abs(F2))
                 + U * np.where(_sterbenz(S[1], S[0]), 0.0, np.abs(F1)) + 6 * U * lam
                 + eps[idx[0]] + 3 * eps[idx[1]] + 3 * eps[idx[2]] + eps[idx[3]]
                 + win[0] + 2 * win[1] + win[2])
        else:
            D1 = (c[idx[1]] - c[idx[0]]).astype(np.float64)
            D2 = (c[idx[2]] - c[idx[0]]).astype(np.float64)
            lam = U * (np.abs(D2) + 2 * np.abs(D1)) + U * (3 * C[0] + 2 * C[1] + C[2])
            e = 2 * U * at + 5 * U * lam + eps[idx[0]] + 2 * eps[idx[1]] + eps[idx[2]] + win[0] + win[1]
        e *= 1.0 + 1e-6
        with np.errstate(over='ignore'):
            esq = float(np.sum(e * (2 * at + e)))
            st2 = float(np.sum(t * t))
        D = 8 + 5 + 8 + -(-self.sq_tiles // 32) + 5           # thread, butterfly, warps, pass-5 lanes, butterfly
        den = (6.0 if self.had else 2.0) * m * m * K
        floor = 2.0 ** -1074 * (1.0 + 2.0 * K / den)            # FMA squares and the division in gradual underflow
        return ((esq + _gamma(D) * (st2 + esq)) * (1 + _gamma(3)) / den + _gamma(3) * st2 / den) * (1 + 1e-6) + floor


def k4o_bound(x, fs, hadamard=False, mult=None, path=None):
    """(var, tau, info, bound): exact() of a series whose samples are finite, with the bound on |K4o - var| of every
    tau (computed from the exact terms)."""
    b = _K4oBound(x, hadamard)
    var, tau, info = exact(x, fs, hadamard, mult, per_tau=b, path=path)
    return var, tau, info, np.array(info['per_tau'])
