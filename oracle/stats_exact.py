"""Exact error statistics: what InsDataMgr.__array_stats computes (np.max(np.abs(x), 0), np.average(x, 0),
np.std(x, 0), ins_data_manager.py:797-808), without the rounding of a float64 reduction.

max|e| is np.max(np.abs(x)) itself (a maximum is exact in any order).  Mean and ddof-0 variance are computed in
integer arithmetic: every float64 is an integer times a power of two, so with X_i = x_i 2^E (E the largest
exponent that makes all of them integers) mean = S / (n 2^E) and std = sqrt(n Q - S^2) / (n 2^E), S = sum X_i,
Q = sum X_i^2.  The mean is rounded once; the square root is taken to ~110 bits with a sticky bit and then
rounded once.

Non-finite samples follow NumPy: a NaN in a column makes its max, mean and std NaN; +-inf makes max inf, mean
+-inf (NaN if both signs occur) and std NaN.  The statistics of no samples are NaN."""
import math

import numpy as np

EPS = np.finfo(np.float64).eps


def _column(v):
    v = [float(a) for a in v]
    n = len(v)
    nan = float('nan')
    if n == 0:
        return nan, nan, nan
    if any(a != a for a in v):
        return nan, nan, nan
    pos, neg = any(a == math.inf for a in v), any(a == -math.inf for a in v)
    if pos or neg:
        return math.inf, (nan if pos and neg else (math.inf if pos else -math.inf)), nan
    mx = max(abs(a) for a in v)
    ratios = [a.as_integer_ratio() for a in v]           # (p, 2^k)
    den = max(q for _, q in ratios)
    X = [p * (den // q) for p, q in ratios]
    S = sum(X)
    Q = sum(x * x for x in X)
    nd = n * den
    mean = S / nd                                        # int / int: correctly rounded
    P = n * Q - S * S                                    # n^2 den^2 var >= 0
    if P == 0:
        return mx, mean, 0.0
    k = max(0, (230 - P.bit_length()) // 2 + 1)
    N = P << (2 * k)
    r = math.isqrt(N)
    r2 = 2 * r + (0 if r * r == N else 1)               # sticky bit: sqrt(N) lies strictly inside (r, r + 1)
    std = r2 / (nd << (k + 1))
    return mx, mean, std


def stats(x, axis=0):
    """[3, ...] = exact (max|x|, mean, std) of x along `axis`, as float64; the other axes keep their shape."""
    x = np.moveaxis(np.asarray(x, dtype=np.float64), axis, 0)
    shape = x.shape[1:]
    flat = x.reshape(x.shape[0], int(np.prod(shape)))
    out = np.array([_column(flat[:, j]) for j in range(flat.shape[1])], dtype=np.float64).T
    return out.reshape((3,) + shape)


def per_run(x, start=0):
    """x [R, n, C] -> [R, 3, C]: exact statistics of every run over samples >= start (the proc_stats layout)."""
    x = np.asarray(x, dtype=np.float64)
    return np.stack([stats(x[r, start:], 0) for r in range(x.shape[0])])


def one_pass_mean_err(x, start):
    """Bound of the rounding of a mean taken in one pass shifted by the first sample (K12, K7) over the samples
    >= start of x [R, n, C] -> [R, C]: the n sequential additions of d = x - x[start] move the sum by at most
    (n - 1) eps sum|d|, the differences and the final division and addition by a few eps more."""
    x = np.asarray(x, dtype=np.float64)[:, start:]
    n = x.shape[1]
    with np.errstate(invalid='ignore'):
        d = np.abs(x - x[:, :1])
    d = np.where(np.isfinite(d), d, 0.0).max(1)
    return (n + 2) * EPS * d + 2 * EPS * np.where(np.isfinite(x), np.abs(x), 0.0).max(1)


def assert_stats(got, ref, mean_err, rel, what='', std_from_mean='second', max_exact=True, abs_slack=0.0):
    """got, ref [..., 3, C] (max, mean, std).  Non-finite reference entries: NaN masks and infinities equal
    exactly.  Finite ones:
      max   equal bit for bit if max_exact (it is the same maximum), else within abs_slack;
      mean  |d| <= mean_err, the caller's bound of the rounding of the mean (e.g. depth eps max|x| for sums
            whose chains of additions are at most `depth` long);
      std   |d| <= rel std + s, rel for the roundings of the squared deviations and s for the error of the
            means they are taken from: std_from_mean 'second': min(m, m^2 / std) with m = mean_err (two
            passes: sqrt(var + m^2) - sqrt(var)); 'first': m (a Chan merge rounds mean_b - mean_a to
            eps max|x|, which moves M2 to first order); 'none': 0 (one shifted pass: the shift has removed
            the offset, rel covers it);
    plus abs_slack on every entry (errors the host recomputes with a different rounding of their own)."""
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    nan_r, nan_g = np.isnan(ref), np.isnan(got)
    assert np.array_equal(nan_r, nan_g), '%s: NaN where NumPy has none at %s, none where it has at %s' % (
        what, np.argwhere(nan_g & ~nan_r)[:5].tolist(), np.argwhere(nan_r & ~nan_g)[:5].tolist())
    inf_r = np.isinf(ref)
    assert np.array_equal(got[inf_r], ref[inf_r]) and not np.isinf(got[~inf_r]).any(), (what, 'infinities')
    fin = np.isfinite(ref)
    mx, mean, sd = np.moveaxis(ref, -2, 0)
    gmx, gmean, gsd = np.moveaxis(got, -2, 0)
    m = np.broadcast_to(np.asarray(mean_err, dtype=np.float64), mean.shape)
    with np.errstate(invalid='ignore', divide='ignore'):
        s = {'second': np.where(sd > 0, np.minimum(m, m * m / sd), m), 'first': m,
             'none': np.zeros_like(m)}[std_from_mean]
        tol = {'max': abs_slack + 0 * sd, 'mean': m + abs_slack, 'std': rel * sd + s + abs_slack}
    for name, g, r in (('max', gmx, mx), ('mean', gmean, mean), ('std', gsd, sd)):
        ok = np.isfinite(r)
        if name == 'max' and max_exact:
            assert np.array_equal(g[ok], r[ok]), '%s: max|e| differs, worst %.3e' % (what, np.abs(g - r)[ok].max())
            continue
        with np.errstate(invalid='ignore'):
            d = np.abs(g - r)
        bad = ok & ~(d <= tol[name])
        assert not bad.any(), '%s %s: %d out of tolerance, worst |d| %.3e at tol %.3e' % (
            what, name, bad.sum(), d[bad].max(), tol[name][bad][np.argmax(d[bad])])
    return fin
