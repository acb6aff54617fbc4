"""The Welch PSD (welch_np's formula) to better than float64 by three orders, the reference of K11; K11's
algorithm restated in float64 (emulate); a rigorous per-bin bound on K11's rounding (the `bound` of
`welch`); and the sharp scale U_k the GPU tests hold K11 to.

Reference.  The segment mean is exact: the samples are integers on the series' lowest exponent
(allan_exact._exponent/_ints), a segment's sum is an integer, and the mean sum/N is carried as three float64
(hi + mid + lo, 159 bits), so y_m = ((x_m - hi) - mid) - lo is formed in np.longdouble (64-bit significand)
to within 2^-62 |y_m| of the exact detrended sample, and no x - mean is ever formed in float64.  Each
segment's real DFT is pocketfft's in long double (bin error ~2e-19 ||y||_2), and |X|^2, the c_k weights, the
segment mean, the scale 1/(fs sum w^2) are long double too; the result is rounded once to float64: +inf where
it exceeds DBL_MAX, subnormal where it is.  A NaN or +-inf inside a used segment makes every bin NaN; samples
past the last segment are never read; finite samples never give NaN.

U_k.  The size of a u-relative rounding (u = 2^-53) spread over each segment, plus one rounding of the
result:
    U_k = scale (1/K) sum_j c_k (2 |X_jk| + d_jk) d_jk  +  u P_k,
    d_jk = u (||y_j||_2 sqrt(log2 P) + u |W_k| ||x_j||_1 / N),    scale = 1 / (fs sum w^2)
so its first-order part is u scale (1/K) sum_j c_k 2 |X_jk| ||y_j||_2 sqrt(log2 P) and d^2 is second order: no
floor in proportion to the segment's power.
X_jk the exact DFT of segment j, W_k the DFT of the window, P the transform length (M on the radix-2 path,
the Bluestein length otherwise).  The second term of d is what the compensated mean (hi + lo) leaves: u^2
|mean| times the window's spectrum.  U_k, the bound and 'segmax' are long double, so they stay finite where
|X|^2 exceeds DBL_MAX.

Bound.  |K11_k - P_k| <= bound_k, with, per segment j and bin k, D_jk >= |X^_jk - X_jk|:
    D_jk = dm_j |W_k| + g3 sum_m |y_m| + g3 2 dh_j sum |w| + F ||y_j||_2
  * dm_j >= |hi + lo - mean|: the residual sum's rounding, g_(d+3) (||x - mean||_1 + g_(d+1) ||x||_1) / N,
    d = ceil(M / gsz) + log2(min(gsz, 32)) + gsz / 32 the depth of K11's mean sum (strided per-thread sums,
    then welch_group_sum's tree); dh_j = g_(d+1) ||x||_1 / N >= |hi - mean|;
  * g3 (|x_m - mean| + 2 dh) |w_m|: the subtraction pair and the window product;
  * F ||y||_2 >= |dX_k| from the transform (Higham, Accuracy and Stability, Thm 24.2: a radix-2 transform of
    length P with twiddles within mu has ||dY||_2 <= log2(P) eta / (1 - log2(P) eta) ||Y||_2, eta = mu +
    g4 (sqrt 2 + mu); mu = 4u covers sincospi and the half-step product), and for |X_k| <= sqrt(M) ||y||_2:
      radix-2:   F = 2 e(M) sqrt(M) + (mu + g5) 2 sqrt(M)          (the transform, then the split step)
      Bluestein: the chirp product (mu + g3), the first transform, bhat's own transform error
                 (sqrt(P (2M - 1)) (mu + e(P))), the pointwise product (g3 with |bhat|_inf), the second
                 transform, the output chirp (mu + g2), divided by P, then the split step as above;
  * |.|^2 of the computed X: g2;
  * the sum over the K segments: depth ceil(Q / G) in a chunk, log2 G for the slot tree and nchunk for
    welch_finish_kernel, and the scale (sum w^2 over 512 threads, fs, K, c): g_R, R = that depth +
    ceil(N / 512) + 9 + 5;
    bound_k = (1 + g_R) scale (1/K) sum_j c_k ((2 |X_jk| + D_jk) D_jk + g2 (|X_jk| + D_jk)^2) + g_R P_k.
The bound assumes no intermediate underflows (every test magnitude is >= 1e-150).

Emulation.  `emulate` runs K11's algorithm in float64 in the kernel's order: the compensated mean over the
strided per-thread sums and the group tree; the bit-reversed radix-2 DIT; the Bluestein pipeline on conj z with
K5's chirp (k^2 reduced mod 2M), bhat made by the same DIT, the DIF back; the split step; the power-of-two
prescales of the mean's summands, y and the powers; the G-slot xor tree and the chunk order.  Its twiddles
and chirps are correctly rounded and its FMAs are plain multiply-adds, so it is not K11's bits; it shows on the CPU that the bound holds, fixes the
sharp thresholds and lets a mistake be tried without a GPU.
"""
import math
from fractions import Fraction

import numpy as np

from allan_exact import _exponent, _ints

LD = np.longdouble
U = 2.0 ** -53
THREADS = 512
CHUNK_SAMPLES = 1 << 18


def have_long_double():
    """True where np.longdouble carries a 64-bit significand, as the reference needs."""
    return np.finfo(np.longdouble).nmant >= 63


def _g(n):
    return n * U / (1.0 - n * U)


def plan(n, N, D):
    """K11's shape: dict of N, M, P, logP, G, bluestein, S, K, Q, nchunk (welch_kernel.cuh welch_plan)."""
    M = N // 2
    if M & (M - 1) == 0:
        P, blue = M, False
    else:
        P, blue = 1, True
        while P < 2 * M - 1:
            P <<= 1
    G = min(32, 1024 // P) if P <= 1024 else 1
    S = N - D
    K = (n - D) // S
    rounds = CHUNK_SAMPLES // (G * N)
    Q = G * max(rounds, 1)
    return dict(N=N, M=M, P=P, logP=P.bit_length() - 1, G=G, bluestein=blue, S=S, K=K, Q=Q,
                nchunk=(K + Q - 1) // Q)


def _segment_means(x, N, S, K):
    """The exact mean of each segment as three float64 (hi, mid, lo), and ||x_j||_1 (float64, rounded up)."""
    used = x[:S * (K - 1) + N]
    E = _exponent(used)
    xi = _ints(used, E)
    pre = np.concatenate([[0], np.cumsum(xi)]) if xi.size else np.zeros(1, dtype=object)
    scale = Fraction(2) ** E
    out = np.zeros((K, 3))
    for j in range(K):
        f = Fraction(int(pre[j * S + N] - pre[j * S])) * scale / N
        for i in range(3):
            out[j, i] = float(f)
            f -= Fraction(out[j, i])
    return out


def _window_dft(w):
    return np.abs(np.fft.rfft(np.asarray(w, dtype=LD)))


def _bhat_inf(M, P):
    """max |bhat|: the transform of the wrapped conjugate chirp of length P, in long double."""
    k = np.arange(M, dtype=np.int64)
    ang = np.asarray((k * k) % (2 * M), dtype=LD) * LD(np.pi) / LD(M)
    c = np.cos(ang) - 1j * np.sin(ang)
    b = np.zeros(P, dtype=np.clongdouble)
    b[:M] = c
    b[P - M + 1:] = c[1:][::-1]
    return float(np.abs(np.fft.fft(b)).max())


def _transform_factor(pl):
    """F of the bound: |dX_k| <= F ||y||_2 from the transform and the split step."""
    mu = 4 * U
    M, P = pl['M'], pl['P']

    def e(n):
        lg = max(int(n).bit_length() - 1, 1)
        eta = mu + _g(4) * (math.sqrt(2) + mu)
        return lg * eta / (1 - lg * eta)
    split = (mu + _g(5)) * 2 * math.sqrt(M)
    if not pl['bluestein']:
        return 2 * e(M) * math.sqrt(M) + split
    rp = math.sqrt(P)
    binf = _bhat_inf(M, P) * (1 + 1e-12)
    da = mu + _g(3)                                     # ||da|| / ||y||
    dA = rp * (da + e(P) * (1 + da)) * (1 + e(P))      # ||dA|| / ||y||
    A = rp * (1 + da)                                   # ||A|| / ||y||
    dbh = rp * math.sqrt(2 * M - 1) * (mu + e(P)) * (1 + mu)
    dB = dA * (binf + dbh) + A * dbh + _g(3) * A * (binf + dbh)
    B = A * (binf + dbh)
    dO = rp * dB + e(P) * rp * (B + dB)
    dZ = (dO + (mu + _g(2)) * P * math.sqrt(M) * (1 + 1e-6)) / P
    return 2 * dZ + split


def welch(x, fs, N, D, window, need=('psd',)):
    """Exact PSD of one series ('psd', float64) and, in long double so that they cannot overflow, the PSD before
    its rounding ('psd_ld'), each bin's largest single-segment PSD ('segmax'), and on request U_k ('U') and
    K11's bound ('bound')."""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(window, dtype=np.float64)
    N, D = int(N), int(D)
    pl = plan(x.size, N, D)
    K, S, M = pl['K'], pl['S'], pl['M']
    L = M + 1
    out = {}
    used = x[:S * (K - 1) + N]
    if not np.all(np.isfinite(used)):
        out['psd'] = np.full(L, np.nan)
        out['U'] = out['bound'] = out['segmax'] = np.zeros(L, dtype=LD)
        out['psd_ld'] = np.full(L, np.nan, dtype=LD)
        return out
    means = _segment_means(x, N, S, K)
    wl = w.astype(LD)
    scale = LD(1) / (LD(fs) * np.sum(wl * wl))
    c = np.full(L, 2.0)
    c[0] = c[-1] = 1.0
    W = _window_dft(w)
    sq = LD(math.sqrt(max(pl['logP'], 1)))
    gsz = THREADS // pl['G']
    d = -(-M // gsz) + int(math.log2(min(gsz, 32))) + gsz // 32
    F = LD(_transform_factor(pl)) * LD(1 + 1e-12) if 'bound' in need else LD(0)
    u = LD(U)
    acc, uacc, bacc, smax = [], [], [], []
    idx = np.arange(N)
    aw = np.abs(w).astype(LD)
    up = LD(1 + 1e-15)
    for j0 in range(0, K, 64):
        j1 = min(K, j0 + 64)
        seg = used[(np.arange(j0, j1) * S)[:, None] + idx]
        mh = means[j0:j1]
        yl = (((seg.astype(LD) - mh[:, 0:1]) - mh[:, 1:2]) - mh[:, 2:3])
        yw = yl * wl
        ny = np.sqrt(np.sum(yw * yw, axis=1)) * up
        X = np.fft.rfft(yw, axis=1)
        a2 = X.real * X.real + X.imag * X.imag
        acc.append(np.ascontiguousarray(a2.T).sum(axis=1))
        smax.append(a2.max(axis=0))
        if 'U' in need or 'bound' in need:
            aX = np.sqrt(a2)
            x1 = np.abs(seg).astype(LD).sum(axis=1) * up
        if 'U' in need:
            dU = u * (ny[:, None] * sq + u * W[None, :] * (x1 / N)[:, None])
            uacc.append(((2 * aX + dU) * dU).sum(axis=0))
        if 'bound' in need:
            dev = np.abs(yl) * up                                          # |x_m - mean|
            xm1 = np.abs(seg.astype(LD) - mh[:, 0:1]).sum(axis=1) * up + N * np.abs(LD(1) * mh[:, 1] + mh[:, 2])
            dh = LD(_g(d + 1)) * x1 / N
            dm = LD(_g(d + 3)) * (xm1 + LD(_g(d + 1)) * x1) / N * LD(1 + 4 * U)
            Dj = (dm[:, None] * W[None, :] * LD(1 + 1e-12)
                  + LD(_g(3)) * ((dev * aw).sum(axis=1) + 2 * dh * aw.sum())[:, None]
                  + F * ny[:, None])
            bacc.append(((2 * aX + Dj) * Dj + LD(_g(2)) * (aX + Dj) ** 2).sum(axis=0))
    tot = np.ascontiguousarray(np.stack(acc).T).sum(axis=1)
    pl_ld = LD(1) * c * tot / K * scale
    out['psd_ld'] = pl_ld
    with np.errstate(over='ignore'):
        out['psd'] = pl_ld.astype(np.float64)
    out['segmax'] = c * np.max(smax, axis=0) * scale
    if 'U' in need:
        out['U'] = scale / K * c * np.sum(uacc, axis=0) + u * pl_ld
    if 'bound' in need:
        R = -(-pl['Q'] // pl['G']) + int(math.log2(pl['G'])) + pl['nchunk'] + -(-N // THREADS) + 14
        gR = LD(_g(R))
        out['bound'] = (1 + gR) * scale / K * c * np.sum(bacc, axis=0) + gR * pl_ld
    return out


# ---- K11 in float64 -------------------------------------------------------------------------------------
def _cis(num, den):
    """e^{j pi num / den}, correctly rounded per component (long double then one rounding)."""
    a = np.asarray(num, dtype=LD) * LD(np.pi) / LD(den)
    return np.cos(a).astype(np.float64) + 1j * np.sin(a).astype(np.float64)


def _bitrev(i, bits):
    r = np.zeros_like(i)
    for b in range(bits):
        r |= ((i >> b) & 1) << (bits - 1 - b)
    return r


def _dit(x, tw, P, sign):
    """fft_dit<sign> on rows of x (bit-reversed in, natural out)."""
    half = 1
    while half < P:
        w = tw[np.arange(half) * (P // (2 * half))]
        if sign < 0:
            w = np.conj(w)
        v = x.reshape(x.shape[0], P // (2 * half), 2, half)
        u, t = v[:, :, 0, :].copy(), w * v[:, :, 1, :]
        v[:, :, 0, :] = u + t
        v[:, :, 1, :] = u - t
        half <<= 1
    return x


def _dif(x, tw, P, sign):
    half = P // 2
    while half >= 1:
        w = tw[np.arange(half) * (P // (2 * half))]
        if sign < 0:
            w = np.conj(w)
        v = x.reshape(x.shape[0], P // (2 * half), 2, half)
        u, t = v[:, :, 0, :].copy(), v[:, :, 1, :].copy()
        v[:, :, 0, :] = u + t
        v[:, :, 1, :] = w * (u - t)
        half >>= 1
    return x


def _group_sum(s, gsz):
    """welch_group_sum over rows of s [rows, gsz]: the xor butterfly in each warp, then warp order."""
    lanes = np.arange(gsz)
    o = min(gsz, 32) // 2
    while o > 0:
        s = s + s[:, lanes ^ o]
        o //= 2
    if gsz <= 32:
        return s[:, 0]
    t = s[:, 0].copy()
    for i in range(1, gsz // 32):
        t = t + s[:, 32 * i]
    return t


def _strided_sum(terms, gsz):
    """Per-thread sums of terms [rows, M] over m = lr, lr + gsz, ... in order, then the group tree."""
    rows, M = terms.shape
    pad = -(-M // gsz) * gsz
    t = np.zeros((rows, pad))
    t[:, :M] = terms
    t = t.reshape(rows, pad // gsz, gsz)
    s = np.zeros((rows, gsz))
    for i in range(t.shape[1]):
        s = s + t[:, i, :]
    return _group_sum(s, gsz)


def emulate(x, fs, N, D, window, mutant=None):
    """K11 in float64 in the kernel's order (see the module docstring). mutant: None or the name of a
    deliberate mistake ('mean_ulp', 'half_step_conj', 'chirp_mod_m', 'chunks_reversed', 'no_fma' is the
    emulation itself) to see which checks catch it."""
    x = np.asarray(x, dtype=np.float64)
    w = np.asarray(window, dtype=np.float64)
    pl = plan(x.size, int(N), int(D))
    N, M, P, logP, G, K, Q, S = (pl[k] for k in ('N', 'M', 'P', 'logP', 'G', 'K', 'Q', 'S'))
    nchunk, blue = pl['nchunk'], pl['bluestein']
    L = M + 1
    gsz = THREADS // G
    e = (N - 1).bit_length()
    ms, mdiv = 2.0 ** -e, N * 2.0 ** -e
    qc = (Q - 1).bit_length()
    qn = (nchunk - 1).bit_length() if nchunk > 1 else 0
    cs, ps = 2.0 ** -qc, 2.0 ** -qn
    # welch_prep_kernel
    wp = np.zeros(-(-N // THREADS) * THREADS)
    wp[:N] = w * w
    s = np.zeros((1, THREADS))
    for r in wp.reshape(-1, THREADS):
        s = s + r
    s = _group_sum(s, THREADS)[0]
    f = fs * s
    a = int(math.frexp(f)[1] - 1) if (f > 0 and math.isfinite(f)) else 0
    a = int(a / 2)
    a = max(-500, min(500, a))
    post = 0.5 / P if blue else 0.5
    with np.errstate(over='ignore', divide='ignore'):
        wscale = (2.0 ** (2 * a + 8) / (cs * ps)) / (float(K) * f)
    cw = (int((math.frexp(s)[1] - 1) / 2) if (s > 0 and math.isfinite(s)) else 0) + 5 + (3 * logP if blue else 0)
    g = math.ldexp(post, e + cw - a - 4)
    ws = w * 2.0 ** -cw
    # tables
    tw = _cis(2 * np.arange(P // 2), P)
    half_step = _cis(-1, M)
    m = np.arange(M)
    chm = M if mutant == 'chirp_mod_m' else 2 * M
    chirp = _cis((m.astype(np.int64) ** 2) % chm, M)
    brP = _bitrev(np.arange(P), logP)
    if blue:
        bh = np.zeros((1, P), dtype=complex)
        bh[0, brP[m]] = np.conj(chirp)
        bh[0, brP[P - m[1:]]] = np.conj(chirp[1:])
        bhat = _dit(bh, tw, P, -1)[0]
    k = np.arange(L)
    kk = np.where(k == M, 0, k)
    kc = np.where(k == 0, 0, M - k)
    if blue:
        wk = _cis(-k, M)
    else:
        h = k >> 1
        wk = np.where(h < M // 2, np.conj(tw[np.minimum(h, M // 2 - 1)]), -1.0 + 0j)
        hs = np.conj(half_step) if mutant == 'half_step_conj' else half_step
        wk = np.where(k & 1, wk * hs, wk)
    chunks = []
    for c0 in range(0, K, Q):
        c1 = min(K, c0 + Q)
        acc = np.zeros((G, L))
        for jb in range(c0, c1, G):
            js = np.arange(jb, min(c1, jb + G))
            seg = x[(js * S)[:, None] + np.arange(N)]
            u, v = seg[:, 0::2], seg[:, 1::2]
            hi = _strided_sum(u * ms + v * ms, gsz) / mdiv
            lo = _strided_sum((u * ms - hi[:, None] * ms) + (v * ms - hi[:, None] * ms), gsz) / mdiv
            if mutant == 'mean_ulp':
                hi = np.nextafter(hi, np.inf)
            yr = ((u * ms - hi[:, None] * ms) - lo[:, None] * ms) * ws[0::2]
            yi = ((v * ms - hi[:, None] * ms) - lo[:, None] * ms) * ws[1::2]
            z = yr + 1j * yi
            buf = np.zeros((len(js), P), dtype=complex)
            if blue:
                buf[:, brP[m]] = np.conj(z) * chirp
                _dit(buf, tw, P, -1)
                buf *= bhat
                _dif(buf, tw, P, 1)
                Z = np.conj(buf[:, brP[m]] * chirp)
            else:
                buf[:, brP[m]] = z
                Z = _dit(buf, tw, P, -1)
            zk, zc = Z[:, kk], Z[:, kc]
            av = (zk.real + zc.real) + 1j * (zk.imag - zc.imag)
            dv = (zk.real - zc.real) + 1j * (zk.imag + zc.imag)
            t = wk * (dv.imag - 1j * dv.real)
            re = (av.real + t.real) * g
            im = (av.imag + t.imag) * g
            acc[:len(js)] = acc[:len(js)] + (re * re + im * im) * cs
        o = 1
        while o < G:
            acc = acc + acc[np.arange(G) ^ o]
            o <<= 1
        chunks.append(acc[0])
    if mutant == 'chunks_reversed':
        chunks = chunks[::-1]
    if nchunk > 1:
        tot = chunks[0] * ps
        for ch in chunks[1:]:
            tot = tot + ch * ps
    else:
        tot = chunks[0]
    cw = np.where((k == 0) | (k == M), 1.0, 2.0)
    with np.errstate(over='ignore', invalid='ignore'):
        return np.where(cw == 1.0, tot, 2.0 * tot) * wscale
