"""NumPy restatement of the soft- and hard-iron magnetometer calibration (demo_algorithms/mag_calibrate.py,
MagCalibrate() in mag_calibrate_src/src/MagCalibration.c:34-306), in two forms.  Test infrastructure only.

segments: ((x0, xf), (y0, yf), (z0, zf)), half-open row ranges of the rotations about the sensor's x, y and
z axes.  Both forms return (soft_iron [3, 3], hard_iron [4]) and give NaN in all 13 values when a 3x3 or the
4x4 system is singular (solve()).

  * calibrate_direct: the reference's steps on the samples (plane-fit normals, in-place staged corrections,
    sensitivities from ranges, the [2c, 1] / |c|^2 sphere fit), each segment on its own copy of the rows.
  * calibrate_moments: what K10 (gnss_ins_sim_b200/csrc/magcal_kernel.cuh) computes: per-segment moments
    sum d, sum d d^T and the ten cubic monomials of d = m - t (t = the first row of the x segment), the
    normals from the moments shifted back, the ranges from a second pass over the samples, and the sphere
    fit in the shifted calibrated frame u = S d, where the 4x4 system is well conditioned whatever the
    hard iron, equilibrated by a power of two (sphere_scale) so that it is well scaled whatever the units.
    Any non-finite output makes all 13 NaN.
"""
import numpy as np

from oracle_np import normal_pair

# (i, j, k) of the ten cubic monomials, in K10's order
CUBIC = ((0, 0, 0), (0, 0, 1), (0, 0, 2), (0, 1, 1), (0, 1, 2), (0, 2, 2), (1, 1, 1), (1, 1, 2), (1, 2, 2),
         (2, 2, 2))
# (i, j) of the six quadratic monomials
QUAD = ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))
SING_TOL = 1e-12     # a pivot at or below SING_TOL * max|A| makes the system singular


def check_segments(segments, n):
    """The segments as a (3, 2) int64 array; ValueError unless each is a half-open range of >= 3 rows
    inside [0, n)."""
    try:
        seg = np.array(segments, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError('segments must be ((x0, xf), (y0, yf), (z0, zf))')
    if seg.shape != (3, 2) or not np.all(np.isfinite(seg)) or not np.all(seg == np.floor(seg)):
        raise ValueError('segments must be three (start, end) pairs of integer row indices')
    seg = seg.astype(np.int64)
    for a, b in seg:
        if a < 0 or b > n or b - a < 3:
            raise ValueError('segment (%d, %d) must hold at least 3 rows inside [0, %d)' % (a, b, n))
    return seg


def solve(A, b):
    """A x = b by Gaussian elimination with partial pivoting (K10's order of operations); all-NaN x when a
    pivot is at or below SING_TOL * max|A| (or A holds a NaN)."""
    A = np.array(A, dtype=np.float64)
    x = np.array(b, dtype=np.float64)
    n = len(x)
    amax = np.max(np.abs(A))
    for c in range(n):
        p = c + int(np.argmax(np.abs(A[c:, c])))
        if not abs(A[p, c]) > SING_TOL * amax:
            return np.full(n, np.nan)
        if p != c:
            A[[c, p]] = A[[p, c]]
            x[[c, p]] = x[[p, c]]
        for r in range(c + 1, n):
            f = A[r, c] / A[c, c]
            A[r, c:] -= f * A[c, c:]
            x[r] -= f * x[c]
    for c in range(n - 1, -1, -1):
        x[c] = (x[c] - A[c, c + 1:].dot(x[c + 1:])) / A[c, c]
    return x


def _normal(v):
    """The reference's sign rule (largest-magnitude component positive) and normalisation."""
    i = int(np.argmax(np.abs(v)))
    if v[i] < 0.0:
        v = -v
    return v / np.sqrt(v.dot(v))


def _sens(rx, ry, rz):
    """s from the ranges: rx = (range c_z, range c_y) on the x segment, ry = (range c_z, range c_x) on the y
    segment, rz = (range c_y, range c_x) on the z segment (MagCalibration.c:118-148)."""
    sZ2Y, sZ2X, sY2X = rx[0] / rx[1], ry[0] / ry[1], rz[0] / rz[1]
    return np.array([1.0, 1.0 / sY2X, (1.0 + sY2X * sY2X) / (sY2X * sY2X * sZ2X + sY2X * sZ2Y)])


_RANGE_COLS = ((2, 1), (2, 0), (1, 0))     # the two calibrated columns whose ranges each segment gives


def _ranges(c, k):
    a, b = _RANGE_COLS[k]
    return (c[:, a].max() - c[:, a].min(), c[:, b].max() - c[:, b].min())


def _nan_result(segs):
    return np.full((3, 3), np.nan), np.full(4, np.nan)


def _inv_solve(A, b):
    """inv(A) b, as the reference solves (mtxInverse, then a product); all-NaN when A is exactly singular or
    holds a NaN.  No threshold: the reference's own 4x4 system is ill conditioned at large hard iron."""
    try:
        return np.linalg.inv(A).dot(b)
    except np.linalg.LinAlgError:
        return np.full(len(b), np.nan)


def calibrate_direct(mag, segments):
    """MagCalibrate on the rows of mag [n, 3]; also returns mag_cal [sum of lengths, 3], the segments after
    the staged corrections O m, diag(s) ., - hard_iron[0:3]."""
    mag = np.asarray(mag, dtype=np.float64)
    seg = check_segments(segments, mag.shape[0])
    segs = [mag[a:b].copy() for a, b in seg]
    normals = []
    for m in segs:
        v = _inv_solve(m.T.dot(m), m.sum(0))
        normals.append(_normal(v))
    O = np.array(normals)
    segs = [m.dot(O.T) for m in segs]
    s = _sens(*(_ranges(c, k) for k, c in enumerate(segs)))
    S = np.diag(s).dot(O)
    segs = [c * s for c in segs]
    c = np.concatenate(segs)
    H = np.concatenate([2.0 * c, np.ones((c.shape[0], 1))], axis=1)
    p = _inv_solve(H.T.dot(H), H.T.dot((c * c).sum(1)))
    hi = np.array([p[0], p[1], p[2], np.sqrt(p[3] + p[0:3].dot(p[0:3]))])
    if np.isnan(O).any() or np.isnan(p).any():
        S, hi = _nan_result(seg)
    return S, hi, c - hi[0:3]


THREADS = 256      # K10's CTA: thread j sums rows j, j + 256, ... of a segment, then 8 warps of 32 lanes


def _kernel_sum(x):
    """The column sums of x [L, K] in K10's order: per thread at stride THREADS, the xor butterfly within each
    warp (lane l adds lane l ^ o, o = 16 .. 1), then the warps in order."""
    L, K = x.shape
    rounds = -(-L // THREADS)
    xp = np.zeros((rounds * THREADS, K))
    xp[:L] = x
    xp = xp.reshape(rounds, THREADS, K)
    acc = np.zeros((THREADS, K))
    for i in range(rounds):
        acc = acc + xp[i]
    v = acc.reshape(THREADS // 32, 32, K)
    lane = np.arange(32)
    o = 16
    while o:
        v = v + v[:, lane ^ o]
        o >>= 1
    s = v[0, 0].copy()
    for w in range(1, THREADS // 32):
        s = s + v[w, 0]
    return s


def moments(mag, seg, t, order='numpy'):
    """Per segment: count, sum d [3], sum d d^T [6] (QUAD), cubic sums [10] (CUBIC) of d = m - t; the sums in
    NumPy's order, or in K10's (order='kernel', _kernel_sum)."""
    out = []
    for a, b in seg:
        d = mag[a:b] - t
        q = np.stack([d[:, i] * d[:, j] for i, j in QUAD], axis=1)
        cub = np.stack([q[:, QUAD.index((i, j))] * d[:, k] for i, j, k in CUBIC], axis=1)
        if order == 'kernel':
            s = _kernel_sum(np.concatenate([d, q, cub], axis=1))
            out.append((b - a, s[0:3], s[3:9], s[9:19]))
        else:
            out.append((b - a, d.sum(0), q.sum(0), cub.sum(0)))
    return out


def sym3(q):
    """[6] (QUAD) -> symmetric [3, 3]."""
    M = np.empty((3, 3))
    for v, (i, j) in zip(q, QUAD):
        M[i, j] = M[j, i] = v
    return M


def cubic_tensor(cub):
    """[10] (CUBIC) -> symmetric [3, 3, 3]."""
    T = np.empty((3, 3, 3))
    for v, (i, j, k) in zip(cub, CUBIC):
        for a, b, c in {(i, j, k), (i, k, j), (j, i, k), (j, k, i), (k, i, j), (k, j, i)}:
            T[a, b, c] = v
    return T


def sphere_scale(tr, N):
    """(f, e): f = 2^-e, e = floor((e_tr - e_N) / 2) from the binary exponents (frexp) of tr = trace(sum u u^T)
    and N, so f is within a factor 2 of 1 / rms |u|; e = 0 unless tr is finite and positive.  K10 fits the sphere
    to f u, which puts every entry of its 4x4 system on the scale of N."""
    if not (np.isfinite(tr) and tr > 0.0):
        return 1.0, 0
    e = (int(np.frexp(tr)[1]) - int(np.frexp(float(N))[1])) >> 1
    return np.ldexp(1.0, -e), e


def calibrate_moments(mag, segments, order='numpy'):
    """K10's formulation (module docstring): soft_iron [3, 3], hard_iron [4].  order='kernel' sums the moments
    in K10's order (_kernel_sum); the rest already follows K10's order of operations."""
    mag = np.asarray(mag, dtype=np.float64)
    seg = check_segments(segments, mag.shape[0])
    t = mag[seg[0, 0]].copy()
    with np.errstate(all='ignore'):
        mom = moments(mag, seg, t, order)
        normals = []
        for N, s1, q, _ in mom:
            A = sym3(q) + np.outer(t, s1) + np.outer(s1, t) + N * np.outer(t, t)
            normals.append(_normal(solve(A, s1 + N * t)))
        O = np.array(normals)
        s = _sens(*(_ranges(mag[a:b].dot(O.T), k) for k, (a, b) in enumerate(seg)))
        S = np.diag(s).dot(O)
        N = float(sum(m[0] for m in mom))
        D = [(mom[0][i] + mom[1][i]) + mom[2][i] for i in (1, 2, 3)]
        D1, D2, D3 = D[0], sym3(D[1]), cubic_tensor(D[2])
        U1 = S.dot(D1)
        U2 = S.dot(D2).dot(S.T)
        # sum u_i |u|^2 = (S w)_i with w_a = sum_bc (S^T S)_bc D3_abc
        w = np.einsum('bc,abc->a', S.T.dot(S), D3)
        tr = (U2[0, 0] + U2[1, 1]) + U2[2, 2]
        f, _ = sphere_scale(tr, N)
        f2 = f * f
        HH = np.empty((4, 4))
        HH[0:3, 0:3] = (4.0 * U2) * f2
        HH[0:3, 3] = HH[3, 0:3] = (2.0 * U1) * f
        HH[3, 3] = N
        HB = np.append((2.0 * S.dot(w)) * (f2 * f), tr * f2)
        q = solve(HH, HB)
        q[0:3] /= f
        q[3] /= f2
        T = S.dot(t)
        hi = np.array([q[0] + T[0], q[1] + T[1], q[2] + T[2], np.sqrt(q[3] + q[0:3].dot(q[0:3]))])
    if np.isnan(O).any() or np.isnan(q).any() or not (np.isfinite(S).all() and np.isfinite(hi).all()):
        return _nan_result(seg)
    return S, hi


def apply(mag, segments, soft_iron, hard_iron):
    """mag_cal: the segments stacked, each row S m - hard_iron[0:3]."""
    seg = check_segments(segments, np.asarray(mag).shape[0])
    m = np.concatenate([np.asarray(mag)[a:b] for a, b in seg])
    return m.dot(np.asarray(soft_iron).T) - np.asarray(hard_iron).reshape(-1)[0:3]


def calibration_error(soft_iron, hard_iron, si, hi, b):
    """[13]: E = S si / k - I (9, row-major), hard_iron[0:3] / k - hi (3), hard_iron[3] / k - b (1), with
    k = trace(S si) / 3 and b = |ref_mag[0]|."""
    P = np.asarray(soft_iron).dot(np.asarray(si))
    k = np.trace(P) / 3.0
    hard_iron = np.asarray(hard_iron).reshape(-1)
    return np.concatenate([(P / k - np.eye(3)).reshape(-1), hard_iron[0:3] / k - np.asarray(hi),
                           [hard_iron[3] / k - b]])


# ---- synthetic inputs, rebuilt from the recipe tests/golden/magcal.npz stores -----------------------------------
SYN_ROTATIONS, SYN_PLANE, SYN_PLANE_NAN, SYN_PLANE_CONST = 0, 1, 2, 3
SYN_SEED = 2026
QUANTUM = 2.0 ** -24     # uT: inputs are rounded to it, so an ulp of a platform's cos / log cannot change them


def quantize(x):
    return np.round(np.asarray(x) / QUANTUM) * QUANTUM


def synthetic_mag(shape, ns, noise=0.0, b=None, si=None, hi=None, run=0):
    """The samples [sum(ns), 3] of one synthetic case.  SYN_ROTATIONS: rotations of the field b about x, y and z
    (396 degrees each, ns[k] samples), measured as (b_rot + hi) si^T + noise z, z the Philox normals of
    (sample, 13 / 14, run) under SYN_SEED.  SYN_PLANE*: noise-free circles of radius 40 uT in the planes
    x = 0, y = 1 and z = 5 (ns[0] samples each); _NAN shifts x by 10 uT and makes one sample NaN, _CONST shifts
    x by 10 uT and holds the y segment constant."""
    if shape == SYN_ROTATIONS:
        rows = []
        k0 = 0
        for ax, n in enumerate(ns):
            ang = np.linspace(0.0, 2.2 * np.pi, int(n))
            c, s = np.cos(ang), np.sin(ang)
            i, j = [(1, 2), (2, 0), (0, 1)][ax]
            bb = np.tile(np.asarray(b, dtype=np.float64), (int(n), 1))
            bb[:, i], bb[:, j] = c * b[i] + s * b[j], -s * b[i] + c * b[j]
            k = np.arange(k0, k0 + int(n), dtype=np.uint64)
            z = np.empty((int(n), 3))
            z[:, 0], z[:, 1] = normal_pair(k, 13, np.uint64(run), SYN_SEED)
            z[:, 2], _ = normal_pair(k, 14, np.uint64(run), SYN_SEED)
            rows.append((bb + hi).dot(np.asarray(si).T) + noise * z)
            k0 += int(n)
        return quantize(np.concatenate(rows))
    n = int(ns[0])
    ang = np.linspace(0.0, 7.0, n)
    mag = np.concatenate([np.stack([np.zeros(n), 40 * np.cos(ang), 40 * np.sin(ang)], 1),
                          np.stack([40 * np.cos(ang) + 3, np.ones(n), 40 * np.sin(ang)], 1),
                          np.stack([40 * np.cos(ang) + 3, 40 * np.sin(ang) + 1, np.full(n, 5.0)], 1)])
    if shape != SYN_PLANE:
        mag[:, 0] += 10.0
    if shape == SYN_PLANE_NAN:
        mag[n + 17, 1] = np.nan
    if shape == SYN_PLANE_CONST:
        mag[n:2 * n] = mag[n]
    return quantize(mag)


def golden_synthetic(g, i):
    """(mag, segments, kind) of synthetic case i of tests/golden/magcal.npz, rebuilt from its recipe."""
    p = lambda k: g['syn%d_%s' % (i, k)]     # noqa: E731
    mag = synthetic_mag(int(p('shape')), p('ns'), float(p('noise')), p('b'), p('si'), p('hi'), int(p('run')))
    return mag, p('seg'), int(p('kind'))
