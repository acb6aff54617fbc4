"""Exact references for the device's FP64 primitives (csrc/fastmath64.cuh, mech.cuh's sincos_angle) and
for the Box-Muller normals of the noise generator (common.cuh normal_from_words).

Errors are measured in ulps of the exact result.  The reference is np.longdouble (a 64-bit significand on
x86-64: 11 bits beyond float64, so a result is known to ~5e-4 ulp); `have_long_double()` says whether this
platform has it.  Where a function is specified against a correctly rounded IEEE operation (1/x, a/b,
sqrt), the points where the device differs from NumPy's correctly rounded result and could hold the largest
error have it computed exactly with Python integers: that is what resolves sqrt_nr's 0.5005-ulp bound.

The hard-case generators give the arguments where these functions go wrong: the doubles nearest every
multiple of pi/2 (tiny reduced arguments), the odd multiples of pi/4 (quadrant flips), binade edges, log's
sqrt(2) switch, and the ends of the Box-Muller domain."""
import math
from fractions import Fraction

import numpy as np

LD = np.longdouble
# pi to 40 digits: exact enough for any Fraction below (2^-130 relative)
PI_STR = '3.141592653589793238462643383279502884197'
PI_FRAC = Fraction(PI_STR)
PI_LD = LD(PI_STR)

# the Cody-Waite split of pi/2 in sincos_bounded (fastmath64.cuh PIO2_1..3)
PIO2_1 = 1.57079632673412561417e+00
PIO2_2 = 6.07710050630396597660e-11
PIO2_3 = 2.02226624871116645580e-21
# |pi/2 - (PIO2_1 + PIO2_2 + PIO2_3)|: the reduction's own error per unit of the quadrant index
PIO2_SPLIT_ERR = float(abs(PI_FRAC / 2 - (Fraction(PIO2_1) + Fraction(PIO2_2) + Fraction(PIO2_3))))
ANGLE_LIMIT = 1.0e6          # mech.cuh sincos_angle: larger magnitudes are taken as the angle 0


def have_long_double():
    return np.finfo(np.longdouble).nmant >= 63


def ulp_of(y):
    """ulp of the float64 format at the exact value(s) y (long double): 2^(e - 52) for 2^e <= |y| < 2^(e+1),
    2^-1074 below the normal range; 0 where y == 0."""
    y = np.abs(np.asarray(y, dtype=LD))
    _, e = np.frexp(y)                        # y = m 2^e, m in [0.5, 1)
    u = np.ldexp(np.ones_like(y), np.maximum(e.astype(np.int64) - 53, -1074))
    return np.where(y == 0, LD(0), u)


def ulp_err(got, want):
    """|got - want| in ulps of want (long double).  An exact zero must be met exactly (0 or inf); two NaNs
    agree."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=LD)
    d = np.abs(got.astype(LD) - want)
    u = ulp_of(want)
    with np.errstate(divide='ignore', invalid='ignore'):
        e = np.where(u > 0, d / np.where(u > 0, u, 1), np.where(d == 0, LD(0), LD(np.inf)))
    both_nan = np.isnan(got) & np.isnan(want)
    return np.where(both_nan, LD(0), np.where(np.isnan(e), LD(np.inf), e)).astype(np.float64)


def ld_fraction(v):
    """The long double v as an exact Fraction."""
    m, e = np.frexp(LD(v))
    return Fraction(int(np.ldexp(m, 64))) * Fraction(2) ** (int(e) - 64)


# ---- exact errors against correctly rounded operations -----------------------------------------------
def _frac_ulp(q):
    """ulp of float64 at the exact nonzero rational q."""
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    return Fraction(2) ** max(e - 52, -1074)


def _exact_err(got, exact):
    return float(abs(Fraction(got) - exact) / _frac_ulp(exact))


def rcp_err(x, got):
    """Exact ulp error of got = 1/x where it can hold the maximum; see _rounded_err."""
    x = np.asarray(x, dtype=np.float64)
    return _rounded_err(got, 1.0 / x, LD(1) / x.astype(LD), lambda i: 1 / Fraction(float(x[i])))


def div_err(a, b, got):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return _rounded_err(got, a / b, a.astype(LD) / b.astype(LD),
                        lambda i: Fraction(float(a[i])) / Fraction(float(b[i])))


def _sqrt_frac_err(x, s):
    """|s - sqrt(x)| / ulp(sqrt(x)) for doubles x > 0 and s, exactly up to 2^-100 ulp: sqrt(x) 2^P lies in
    [lo, lo + 1) with lo = isqrt(floor(x 4^P)) and P chosen so that lo has ~160 bits; the larger of the
    two ends' errors is returned."""
    _, ex = math.frexp(x)
    P = 160 - ex // 2
    scaled = Fraction(x) * Fraction(4) ** P
    lo = math.isqrt(scaled.numerator // scaled.denominator)
    root_lo, root_hi = Fraction(lo) / Fraction(2) ** P, Fraction(lo + 1) / Fraction(2) ** P
    u = _frac_ulp(root_lo)
    fs = Fraction(s)
    return float(max(abs(fs - root_lo), abs(fs - root_hi)) / u)


def sqrt_err(x, got):
    """Exact ulp error of got = sqrt(x) (x >= 0) where it can hold the maximum; sqrt(0) must be exactly 0."""
    x = np.asarray(x, dtype=np.float64)
    got = np.asarray(got, dtype=np.float64)
    err = _rounded_err(got, np.sqrt(x), np.sqrt(x.astype(LD)), lambda i: None,
                       exact_err=lambda i: _sqrt_frac_err(float(x[i]), float(got[i])), zero=x == 0)
    return err


EXACT_SLACK = 2e-3       # the long-double estimate of an error is good to ~5e-4 ulp


def _rounded_err(got, cr, ref_ld, exact_at, exact_err=None, zero=None):
    """Errors in ulps against a correctly rounded operation: at most 0.5 where got is NumPy's correctly
    rounded cr; elsewhere the long-double estimate, replaced by the exact error (Python integers) at every
    point whose estimate is within EXACT_SLACK of the largest, so that the maximum is exact.  zero: points
    whose exact result is 0 (got must be 0 there)."""
    got = np.asarray(got, dtype=np.float64)
    est = ulp_err(got, ref_ld)
    diff = got != np.asarray(cr, dtype=np.float64)
    err = np.where(diff, est, np.minimum(est, 0.5))
    if zero is not None:
        err[zero] = np.where(got[zero] == 0, 0.0, np.inf)
        diff &= ~zero
    if not diff.any():
        return err
    top = err[diff].max()
    if not np.isfinite(top):
        return err
    cand = np.nonzero(diff & (err >= top - EXACT_SLACK))[0]
    for i in cand[np.argsort(-err[cand])][:10000]:
        err[i] = exact_err(i) if exact_err else _exact_err(float(got[i]), exact_at(i))
    return err


# ---- long-double references --------------------------------------------------------------------------
def rsqrt_ref(x):
    return LD(1) / np.sqrt(np.asarray(x, dtype=LD))


def sincos_ref(x):
    """(sin, cos)(x) in long double, evaluated once per distinct |x| (the hard-case sets are symmetric)."""
    x = np.asarray(x, dtype=np.float64)
    a, inv = np.unique(np.abs(x), return_inverse=True)
    a = a.astype(LD)
    s, c = np.sin(a)[inv].reshape(x.shape), np.cos(a)[inv].reshape(x.shape)
    return np.where(np.signbit(x), -s, s), c


def sincos_angle_ref(x):
    """mech.cuh sincos_angle: (sin, cos) of x for |x| <= 1e6, of 0 beyond, NaN for +-inf and NaN."""
    x = np.asarray(x, dtype=np.float64)
    xa = np.where(np.abs(x) <= ANGLE_LIMIT, x, np.where(np.isfinite(x), 0.0, np.nan))
    return sincos_ref(xa)


def sincospi_ref(x):
    """(sin, cos)(pi x) for doubles x in [0, 2): x - q / 2 is exact, so only pi r with |r| <= 1/4 is
    evaluated; the quadrant points are exact."""
    x = np.asarray(x, dtype=np.float64)
    q = np.rint(2.0 * x)
    r = (x - 0.5 * q).astype(LD)              # exact
    sr, cr = np.sin(PI_LD * r), np.cos(PI_LD * r)
    qi = q.astype(np.int64) & 3
    s = np.select([qi == 0, qi == 1, qi == 2], [sr, cr, -sr], -cr)
    c = np.select([qi == 0, qi == 1, qi == 2], [cr, -sr, -cr], sr)
    return s, c


def log_ref(x):
    return np.log(np.asarray(x, dtype=LD))


def box_muller_ref(words):
    """words [n, 4] uint32 (Philox x0..x3) -> (z0*, z1*, r*) in long double from the exact uniforms
    u1 = 1 - m1 2^-52, u2 = m2 2^-52 (m1 = (x1:x0) >> 12, m2 = (x3:x2) >> 12)."""
    w = np.asarray(words, dtype=np.uint64)
    m1 = ((w[:, 1] << np.uint64(32)) | w[:, 0]) >> np.uint64(12)
    m2 = ((w[:, 3] << np.uint64(32)) | w[:, 2]) >> np.uint64(12)
    u1 = LD(1) - m1.astype(LD) * LD(2.0 ** -52)           # exact: 53 bits
    r = np.sqrt(LD(-2) * np.log(u1))
    s, c = sincospi_ref(m2.astype(np.float64) * 2.0 ** -51)   # 2 u2, exact
    return r * c, r * s, r


def words_from_m(m1, m2):
    """Philox outputs whose 52-bit mantissas are m1 (u1) and m2 (u2); the discarded 12 low bits are 0."""
    a = np.asarray(m1, dtype=np.uint64) << np.uint64(12)
    b = np.asarray(m2, dtype=np.uint64) << np.uint64(12)
    a, b = np.broadcast_arrays(a, b)
    lo = np.uint64(0xFFFFFFFF)
    return np.stack([a & lo, a >> np.uint64(32), b & lo, b >> np.uint64(32)], axis=-1).astype(np.uint32)


# ---- hard cases ---------------------------------------------------------------------------------------
def neighbours(x, k):
    """x and its k nearest doubles on each side (flattened)."""
    x = np.asarray(x, dtype=np.float64).ravel()
    out = [x]
    up, dn = x.copy(), x.copy()
    for _ in range(k):
        up = np.nextafter(up, np.inf)
        dn = np.nextafter(dn, -np.inf)
        out += [up, dn]
    return np.concatenate(out)


def halfpi_multiples(limit, k=4):
    """The doubles nearest every k pi/2 with |k pi/2| <= limit, +-4 ulp, both signs: where the reduced
    argument is tiny."""
    n = int(LD(limit) / (PI_LD / 2))
    x = (np.arange(1, n + 1, dtype=LD) * (PI_LD / 2)).astype(np.float64)
    x = neighbours(x[np.abs(x) <= limit], k)
    return np.concatenate([[0.0], x, -x])


def odd_quarterpi_multiples(limit=64.0, k=4):
    """The doubles nearest every odd k pi/4 with |x| <= limit, +-4 ulp, both signs: where the rounding
    trick's quadrant flips and |r| reaches pi/4."""
    n = int(LD(limit) / (PI_LD / 4))
    j = np.arange(1, n + 1, 2, dtype=LD)
    x = neighbours((j * (PI_LD / 4)).astype(np.float64), k)
    x = x[np.abs(x) <= limit]
    return np.concatenate([x, -x])


def binade_edges(lo_exp, hi_exp, k=4):
    """2^e +- k ulp for lo_exp <= e <= hi_exp."""
    return neighbours(np.ldexp(1.0, np.arange(lo_exp, hi_exp + 1)), k)


def log_hard_cases():
    """log_unit on [2^-52, 1]: mantissas within +-8 ulp of sqrt(2) in every binade (the 0x95f64 halving
    switch), the binade edges, and x = 1 - m 2^-52 for small m."""
    sq = np.ldexp(math.sqrt(2.0), np.arange(-53, 0))         # sqrt(2) 2^e in [2^-52, 1)
    x = np.concatenate([neighbours(sq, 8), binade_edges(-52, 0, 8),
                        1.0 - np.arange(0, 4097) * 2.0 ** -52, 1.0 - np.arange(1, 64) * 2.0 ** -40])
    return np.unique(x[(x >= 2.0 ** -52) & (x <= 1.0)])


def sincos_angle_specials():
    big = np.array([ANGLE_LIMIT, np.nextafter(ANGLE_LIMIT, np.inf), np.nextafter(ANGLE_LIMIT, 0.0), 2e6,
                    1e300, np.finfo(np.float64).max])
    return np.concatenate([[0.0, -0.0], big, -big, [np.inf, -np.inf, np.nan]])


# ---- the domains the suite holds each function to, and the bounds ------------------------------------
# ulps of the exact result unless named _ABS.  sincos_bounded / sincos_angle: |err| <= K ulp(result)
# + |q| PIO2_SPLIT_ERR, q the quadrant index.  The three-term split of pi/2 stops at PIO2_3, so the reduced
# argument carries |q| 8.5e-32 absolute: near the zeros of sin and cos that is up to 2.6e4 ulp of the result
# for |x| <= 64 (at the double nearest 29 pi / 2) and 2.8e6 ulp for |x| <= 1e6.  The reduction's two
# roundings add up to an ulp of r, which is two ulps of a result just below a power of two.  K is the
# measured worst case with a little headroom; the arguments are seeded, and the device equals the host build
# bit for bit, so the check is deterministic.
SINCOS_K = 1.6                   # |x| <= 64; measured 1.554 (cos at -14.933548946059105)
SINCOS_ANGLE_K = 2.5             # 64 < |x| <= 1e6; measured 2.390 (at -64073.033369127574)
SINCOSPI_ABS = 3e-16
LOG_ULP = 2.0
SQRT_ULP = 0.5005
RSQRT_ULP = 1.0
RCP_ULP = 1.0
DIV_ULP = 1.0


def quadrant(x):
    """|q| of sincos_bounded's reduction (the nearest integer to x 2 / pi)."""
    return np.abs(np.rint(np.asarray(x, dtype=np.float64) * (2.0 / np.pi)))


def sincos_excess(x, s, c, ref_s, ref_c):
    """max over sin and cos of (|err| - |q| PIO2_SPLIT_ERR) / ulp(result): the K of the bound above."""
    q = LD(PIO2_SPLIT_ERR) * quadrant(x).astype(LD)
    out = []
    for got, ref in ((s, ref_s), (c, ref_c)):
        d = np.abs(np.asarray(got, dtype=np.float64).astype(LD) - ref)
        u = ulp_of(ref)
        with np.errstate(divide='ignore', invalid='ignore'):
            k = np.where(u > 0, (d - q) / np.where(u > 0, u, 1), np.where(d <= q, LD(0), LD(np.inf)))
        out.append(k.astype(np.float64))
    return np.maximum(out[0], out[1])


def sincos_args(n, seed):
    """|x| <= 64: uniform on [-64, 64] and on [-pi, pi], and the hard cases."""
    rng = np.random.default_rng(seed)
    x = np.concatenate([rng.uniform(-64.0, 64.0, n), rng.uniform(-np.pi, np.pi, n), halfpi_multiples(64.0),
                        odd_quarterpi_multiples(64.0), binade_edges(-30, 5)])
    x = np.concatenate([x, -binade_edges(-30, 5)])
    return x[np.abs(x) <= 64.0]


def sincos_angle_args(n, seed):
    """64 < |x| <= 1e6: uniform, every k pi/2 +- 4 ulp, and the binade edges."""
    rng = np.random.default_rng(seed)
    x = np.concatenate([rng.uniform(64.0, ANGLE_LIMIT, n) * rng.choice([-1.0, 1.0], n),
                        halfpi_multiples(ANGLE_LIMIT), binade_edges(6, 19), -binade_edges(6, 19)])
    return x[(np.abs(x) > 64.0) & (np.abs(x) <= ANGLE_LIMIT)]


def sincospi_args(n, seed):
    """x = 2 m 2^-52 (2 u2 of Box-Muller): random m, and m within 64 of the quadrant points."""
    rng = np.random.default_rng(seed)
    m = rng.integers(0, 1 << 52, n, dtype=np.uint64)
    pts = np.array([0, 1 << 50, 1 << 51, 3 << 50, 1 << 52], dtype=np.int64)
    near = (pts[:, None] + np.arange(-64, 65)[None, :]).ravel()
    near = near[(near >= 0) & (near < (1 << 52))].astype(np.uint64)
    return np.concatenate([m, near]).astype(np.float64) * 2.0 ** -51


def log_args(n, seed):
    """[2^-52, 1]: u1 = 1 - m 2^-52 for random m (the Box-Muller argument), log-uniform, and the hard cases."""
    rng = np.random.default_rng(seed)
    x = np.concatenate([1.0 - rng.integers(0, 1 << 52, n, dtype=np.uint64).astype(np.float64) * 2.0 ** -52,
                        np.exp2(rng.uniform(-52.0, 0.0, n)), log_hard_cases()])
    return x[(x >= 2.0 ** -52) & (x <= 1.0)]


def sqrt_args(n, seed):
    """[0, 72.1] (-2 ln u1 of Box-Muller): uniform, log-uniform from -2 ln(1 - 2^-52), the binade edges and 0."""
    rng = np.random.default_rng(seed)
    x = np.concatenate([rng.uniform(0.0, 72.1, n), np.exp2(rng.uniform(np.log2(4.4e-16), np.log2(72.1), n)),
                        binade_edges(-51, 6), [0.0, 72.1, -2.0 * math.log(2.0 ** -52)]])
    return x[(x >= 0.0) & (x <= 72.1)]


def rsqrt_args(n, seed):
    """q = 1 - e^2 sin^2(lat) in [0.9933, 1] (mech.cuh geo_param)."""
    rng = np.random.default_rng(seed)
    x = np.concatenate([rng.uniform(0.9933, 1.0, n), neighbours([1.0, 0.9933], 8)])
    return x[(x >= 0.9933) & (x <= 1.0)]


def rcp_args(n, seed):
    """cos(pitch) and cos(lat) on [6e-17, 1] of both signs (log-uniform and uniform), radii near 6.4e6."""
    rng = np.random.default_rng(seed)
    sgn = rng.choice([-1.0, 1.0], n)
    x = np.concatenate([sgn * np.exp2(rng.uniform(np.log2(6e-17), 0.0, n)), sgn * rng.uniform(0.0, 1.0, n),
                        rng.uniform(6.33e6, 6.41e6, n), binade_edges(-53, 0), -binade_edges(-53, 0)])
    return x[((np.abs(x) >= 6e-17) & (np.abs(x) <= 1.0)) | (x > 1e6)]


def div_args(n, seed):
    """(a, b): gps_kernel's sigma / radius and sigma / radius / cos(lat), and log_unit's f / (2 + f) with
    f = m - 1 for m in [sqrt(1/2), sqrt(2))."""
    rng = np.random.default_rng(seed)
    sig = np.exp2(rng.uniform(-10.0, 7.0, n))
    rad = rng.uniform(6.33e6, 6.41e6, n)
    cl = np.exp2(rng.uniform(np.log2(6e-17), 0.0, n))
    m = rng.uniform(math.sqrt(0.5), math.sqrt(2.0), n)
    f = np.concatenate([m - 1.0, neighbours([math.sqrt(0.5) - 1.0, math.sqrt(2.0) - 1.0, 2.0 ** -52], 8)])
    a = np.concatenate([sig, sig / rad, f])
    b = np.concatenate([rad, cl, 2.0 + f])
    return a, b


def box_muller_bound():
    """B of |z - z*| <= B r* 2^-52, from the primitive bounds: log_unit's LOG_ULP relative error is halved by
    the square root, which adds SQRT_ULP; the angle's cos / sin are off by SINCOSPI_ABS absolute; the
    product r cos adds half an ulp of z; 1e-3 covers second-order terms and the long-double reference."""
    return LOG_ULP / 2 + SQRT_ULP + SINCOSPI_ABS / 2.0 ** -52 + 0.5 + 1e-3
