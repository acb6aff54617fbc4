"""The exact magnetometer calibration (MagCalibrate, MagCalibration.c:34-306), the reference of K10, and a bound on
K10's rounding in its own order of operations.  Test infrastructure only.

calibrate(mag, segments) computes every output exactly and rounds it once to float64:
  * moments: every used sample and t (the x segment's first row) is an integer on the run's lowest exponent
    (allan_exact._ints), so the per-segment moments of d = m - t (sum d, sum d d^T, the ten cubic monomials) are
    Python integers;
  * plane fits: (M^T M) x = M^T 1 in Fraction from the exact moments; the sign rule and the normalisation in
    mpmath at PREC bits;
  * extremes of the two columns of O m per segment: every sample in float64, the candidates within a rigorous
    float margin of the max or min re-evaluated in mpmath;
  * s, S and the sphere fit from the exact moments in mpmath: the fit in the shifted frame u = S d is
    algebraically the reference's fit to c = S m ([2c, 1] p = |c|^2, translated by S t), so this is its value;
  * mag_cal, the staged s_i (O_i m) - hard_i, in long double from the exact S, s and hard iron (within 2^-63 of
    the terms, below any bound by 2^10); err, the generated form's calibration error, from the exact S and hard iron.

cls is one of
  'singular'  a non-finite sample, an exactly singular plane or sphere system, or a zero range: K10 returns NaN;
  'regular'   every relative pivot |p_k| / max|A| of the exact systems, as partial pivoting meets them, is above
              REGULAR (the sphere system at the equilibration f of K10 and at f / 2 and 2 f, since K10 takes f from
              its rounded trace), and the first-order bound is below 1e-3 relative: K10 returns a finite result
              within the bound;
  'band'      anything in between: K10 may return NaN, or a result within the bound.

bound(): |K10 - exact| per output (soft_iron [9], hard_iron [4], err [13], mag_cal rows).  It is first order:
every rounding K10 makes is a perturbation of bounded size, carried to the outputs by the exact Jacobian of the
whole pipeline, taken in mpmath by a forward difference of step 2^-120 of each perturbation at PREC bits:
  * each moment: gamma(n) sum |terms|, n = its summation depth (ceil(L / 256) per thread, 5 butterfly steps, 7
    warp additions, 2 segment additions) plus the 1 (sum d), 3 (sum d d^T) or 5 (cubic) roundings of a term;
  * each solve: the formation error of the system, and Gaussian elimination's componentwise backward error
    gamma(3n) |L||U| (Higham, Thm 9.4), carried to the solution through |A^-1|, on the equilibrated 4x4 system;
  * the normalisation gamma(5) |v|, the extremes gamma(3) max_k sum |O_i| |m_k| (a max is 1-Lipschitz), the
    range ratios gamma(3), S = diag(s) O gamma(7), and the final sums and square root directly;
and SLACK (1.25) times the first-order sum covers the second-order terms while the first-order relative bound
is below 1e-3 (the 'regular' condition).  The bound grows like cond(M^T M) u, as K10's error does.
"""
from fractions import Fraction
import mpmath as mp
import numpy as np

from allan_exact import _exponent, _ints
from magcal_np import check_segments, CUBIC, QUAD, _RANGE_COLS, sphere_scale

PREC = 512
REGULAR = 1e-11
SLACK = 1.25
U = 2.0 ** -53
_EPS = mp.mpf(2) ** -120
THREADS = 256


def gamma(n):
    return n * U / (1.0 - n * U)


def _mp(x):
    return mp.mpf(float(x)) if not isinstance(x, (mp.mpf, int, Fraction)) else (
        mp.mpf(x.numerator) / x.denominator if isinstance(x, Fraction) else mp.mpf(x))


def _pivots(A):
    """Relative pivots |p_k| / max|A| of Gaussian elimination with partial pivoting on A (list of lists of
    exact or mp numbers)."""
    A = [list(r) for r in A]
    n = len(A)
    amax = max(abs(v) for r in A for v in r)
    if amax == 0:
        return [0.0] * n
    out = []
    for c in range(n):
        p = max(range(c, n), key=lambda r: abs(A[r][c]))
        out.append(abs(A[p][c]) / amax)
        if A[p][c] == 0:
            return out + [0] * (n - c - 1)
        A[c], A[p] = A[p], A[c]
        for r in range(c + 1, n):
            f = A[r][c] / A[c][c]
            for j in range(c, n):
                A[r][j] -= f * A[c][j]
    return out


def _lu_abs(A):
    """|L||U| of A under partial pivoting (mp), in A's own row order."""
    n = A.rows
    P = list(range(n))
    W = A.copy()
    L = mp.zeros(n, n)
    for c in range(n):
        p = max(range(c, n), key=lambda r: abs(W[r, c]))
        if p != c:
            for j in range(n):
                W[c, j], W[p, j] = W[p, j], W[c, j]
                L[c, j], L[p, j] = L[p, j], L[c, j]
            P[c], P[p] = P[p], P[c]
        L[c, c] = 1
        for r in range(c + 1, n):
            f = W[r, c] / W[c, c]
            L[r, c] = f
            for j in range(c, n):
                W[r, j] -= f * W[c, j]
    LU = mp.matrix([[sum(abs(L[i, k]) * abs(W[k, j]) for k in range(n)) for j in range(n)] for i in range(n)])
    out = mp.zeros(n, n)
    for i in range(n):
        for j in range(n):
            out[P[i], j] = LU[i, j]
    return out


def _solve(A, b):
    """A^-1 b (mp matrices) by Gaussian elimination with partial pivoting and no threshold (mpmath's lu_solve
    refuses pivots below an absolute tolerance, which the scaled cases reach)."""
    n = A.rows
    M = [[A[i, j] for j in range(n)] + [b[i, k] for k in range(b.cols)] for i in range(n)]
    for c in range(n):
        p = max(range(c, n), key=lambda r: abs(M[r][c]))
        M[c], M[p] = M[p], M[c]
        for r in range(c + 1, n):
            f = M[r][c] / M[c][c]
            M[r] = [x - f * y for x, y in zip(M[r], M[c])]
    X = mp.zeros(n, b.cols)
    for k in range(b.cols):
        for c in range(n - 1, -1, -1):
            X[c, k] = (M[c][n + k] - sum(M[c][j] * X[j, k] for j in range(c + 1, n))) / M[c][c]
    return X


def _inv(A):
    return _solve(A, mp.eye(A.rows))


def _absmat(A):
    return mp.matrix([[abs(A[i, j]) for j in range(A.cols)] for i in range(A.rows)])


def _moments(D):
    """Exact integer moments [19] (sum d, QUAD, CUBIC) of the integer rows D [L, 3]."""
    d = [D[:, 0], D[:, 1], D[:, 2]]
    s1 = [int(x.sum()) for x in d]
    q = {ij: d[ij[0]] * d[ij[1]] for ij in QUAD}
    return s1 + [int(q[ij].sum()) for ij in QUAD] + [int((q[(a, b)] * d[c]).sum()) for a, b, c in CUBIC]


def _sym3(q):
    M = mp.zeros(3, 3)
    for v, (i, j) in zip(q, QUAD):
        M[i, j] = M[j, i] = v
    return M


def _cubic(cub):
    T = {}
    for v, (i, j, k) in zip(cub, CUBIC):
        for a, b, c in ((i, j, k), (i, k, j), (j, i, k), (j, k, i), (k, i, j), (k, j, i)):
            T[(a, b, c)] = v
    return T


class _Pipeline:
    """The calibration from the exact moments, the fixed sign choices and the samples at the extremes, with
    an additive perturbation at every place K10 rounds: F(delta) -> (S [9], hard [4], O [9], s [3])."""

    def __init__(self, mom, Ns, t, signs, ext_rows):
        self.mom, self.Ns, self.t, self.signs, self.ext_rows = mom, Ns, t, signs, ext_rows

    def run(self, key=None, val=None):
        d = lambda k, i: val if (k, i) == key else 0      # noqa: E731
        t = self.t
        mom = [[self.mom[s][i] + d('mom', 19 * s + i) for i in range(19)] for s in range(3)]
        O = mp.zeros(3, 3)
        for s in range(3):
            N = self.Ns[s]
            s1, q = mom[s][0:3], mom[s][3:9]
            Q = _sym3(q)
            A = mp.matrix([[Q[i, j] + t[i] * s1[j] + s1[i] * t[j] + N * t[i] * t[j] for j in range(3)]
                           for i in range(3)])
            x = _solve(A, mp.matrix([s1[i] + N * t[i] for i in range(3)]))
            x = [x[i] + d('x', 3 * s + i) for i in range(3)]
            nrm = mp.sqrt(sum(v * v for v in x))
            for i in range(3):
                O[s, i] = self.signs[s] * x[i] / nrm + d('v', 3 * s + i)
        if self.ext_rows is None:
            self.last = dict(O=O)
            return None
        ext = []
        for s in range(3):
            a, b = _RANGE_COLS[s]
            e = []
            for col, rows in ((a, self.ext_rows[s][0:2]), (b, self.ext_rows[s][2:4])):
                for j, m in enumerate(rows):
                    e.append(sum(O[col, i] * m[i] for i in range(3)) + d('ext', 4 * s + 2 * (col == b) + j))
            ext.append(e)
        r = [((ext[s][0] - ext[s][1]) / (ext[s][2] - ext[s][3])) * (1 + d('r', s)) for s in range(3)]
        sZ2Y, sZ2X, sY2X = r
        sv = [mp.mpf(1), 1 / sY2X, (1 + sY2X * sY2X) / (sY2X * sY2X * sZ2X + sY2X * sZ2Y)]
        S = mp.matrix([[sv[i] * O[i, j] + d('Sm', 3 * i + j) for j in range(3)] for i in range(3)])
        N = sum(self.Ns)
        Dm = [mom[0][i] + mom[1][i] + mom[2][i] for i in range(19)]
        D1 = mp.matrix(Dm[0:3])
        D2 = _sym3(Dm[3:9])
        T3 = _cubic(Dm[9:19])
        U1 = S * D1
        U2 = S * D2 * S.T
        G = S.T * S
        w = mp.matrix([sum(G[b, c] * T3[(a, b, c)] for b in range(3) for c in range(3)) for a in range(3)])
        v = S * w
        HH = mp.zeros(4, 4)
        for i in range(3):
            for j in range(3):
                HH[i, j] = 4 * U2[i, j]
            HH[i, 3] = HH[3, i] = 2 * U1[i]
        HH[3, 3] = N
        rhs = mp.matrix([2 * v[0], 2 * v[1], 2 * v[2], U2[0, 0] + U2[1, 1] + U2[2, 2]])
        p = _solve(HH, rhs)
        p = [p[i] + d('q', i) for i in range(4)]
        Tt = S * mp.matrix(t)
        hard = [p[i] + Tt[i] for i in range(3)] + [mp.sqrt(p[3] + p[0] ** 2 + p[1] ** 2 + p[2] ** 2)]
        self.last = dict(HH=HH, rhs=rhs, p=p, S=S, D=Dm, U1=U1, U2=U2, G=G, w=w, v=v, sv=sv, O=O, r=r,
                         ext=ext, tr=U2[0, 0] + U2[1, 1] + U2[2, 2])
        return [S[i, j] for i in range(3) for j in range(3)] + hard + [O[i, j] for i in range(3) for j in range(3)] + sv


def _f64(x):
    return float(x) if mp.isfinite(x) else np.nan


def calibrate(mag, segments, want_bound=True, want_cal=False, model=None):
    """The exact calibration of mag [n, 3] (module docstring).  Returns a dict: cls, soft_iron [3, 3],
    hard_iron [4] (float64, rounded once), pivot (the smallest relative pivot), and with want_bound the bounds
    b_soft [3, 3], b_hard [4], rel (the first-order bound relative to |S| and |hard|); with want_cal mag_cal
    [L, 3] and b_cal [L, 3]; with model = (si, hi, b) err [13] and b_err [13]."""
    with mp.workprec(PREC):
        return _calibrate(np.asarray(mag, dtype=np.float64), segments, want_bound, want_cal, model)


def _calibrate(mag, segments, want_bound, want_cal, model):
    seg = check_segments(segments, mag.shape[0])
    L = sum(int(b - a) for a, b in seg)
    nan = dict(cls='singular', soft_iron=np.full((3, 3), np.nan), hard_iron=np.full(4, np.nan), pivot=0.0,
               err=np.full(13, np.nan), mag_cal=np.full((L, 3), np.nan))
    rows = np.concatenate([mag[a:b] for a, b in seg])
    t_f = mag[seg[0, 0]]
    if not (np.isfinite(rows).all() and np.isfinite(t_f).all()):
        return nan
    E = _exponent(np.concatenate([rows.reshape(-1), t_f]))
    ti = _ints(t_f, E)
    scale = mp.mpf(2) ** E
    t = [mp.mpf(int(v)) * scale for v in ti]
    mom_i, Ns, A_exact, pivots = [], [], [], []
    for a, b in seg:
        Mi = _ints(mag[a:b].reshape(-1), E).reshape(-1, 3)
        mom_i.append(_moments(Mi - ti[None, :]))
        Ns.append(int(b - a))
        # the plane system on m itself, exact: sum m m^T x = sum m
        s1 = [int(Mi[:, i].sum()) for i in range(3)]
        A = [[Fraction(int((Mi[:, i] * Mi[:, j]).sum())) for j in range(3)] for i in range(3)]
        A_exact.append((A, s1))
        pivots += [float(p) for p in _pivots(A)]
    if min(pivots) == 0:
        return dict(nan, pivot=0.0)
    # the normals: x = A^-1 sum m (Fraction), O row = sign * x / |x|; x is in units of 2^-E
    signs, O_f = [], np.empty((3, 3))
    for s, (A, s1) in enumerate(A_exact):
        x = _fsolve(A, [Fraction(v) for v in s1])
        im = max(range(3), key=lambda i: abs(x[i]))
        signs.append(-1 if x[im] < 0 else 1)
        xm = [_mp(v) for v in x]
        nrm = mp.sqrt(sum(v * v for v in xm))
        O_f[s] = [float(signs[s] * v / nrm) for v in xm]
    mom = [[mp.mpf(v) * scale ** (1 if i < 3 else 2 if i < 9 else 3) for i, v in enumerate(m)] for m in mom_i]
    # the extremes: float candidates within a rigorous margin, re-evaluated exactly with the exact O
    pipe = _Pipeline(mom, Ns, t, signs, None)
    pipe.run()
    Oe = pipe.last['O']
    ext_rows, ext_abs = [], []
    for s, (a, b) in enumerate(seg):
        m = mag[a:b]
        er, ea = [], []
        for col in _RANGE_COLS[s]:
            c = m.dot(O_f[col])
            absc = np.abs(m).dot(np.abs(O_f[col]))
            margin = 8 * U * absc.max() * 2
            for pick, sign in ((np.argmax, 1), (np.argmin, -1)):
                ref = c[pick(c)]
                cand = np.nonzero(sign * (c - ref) >= -2 * margin)[0]
                vals = [(sum(Oe[col, i] * mp.mpf(float(m[k, i])) for i in range(3)), k) for k in cand]
                best = max(vals, key=lambda z: sign * z[0])
                er.append([mp.mpf(float(v)) for v in m[best[1]]])
            ea.append(absc.max())
        ext_rows.append(er)
        ext_abs.append(ea)
    pipe.ext_rows = ext_rows
    try:
        base = pipe.run()
    except ZeroDivisionError:       # a zero range
        return dict(nan, pivot=0.0)
    P = pipe.last
    # the sphere system's relative pivots at K10's equilibration and its neighbours
    f, _ = sphere_scale(float(P['tr']), float(sum(Ns)))
    sp = []
    for ff in (f / 2, f, 2 * f):
        Hf = P['HH'].copy()
        for i in range(3):
            for j in range(3):
                Hf[i, j] *= ff * ff
            Hf[i, 3] *= ff
            Hf[3, i] *= ff
        sp.append(min(_pivots([[Hf[i, j] for j in range(4)] for i in range(4)])))
    piv = min(min(pivots), *sp)
    if piv < 1e-60:
        return dict(nan, pivot=0.0)
    out = dict(soft_iron=np.array([_f64(v) for v in base[0:9]]).reshape(3, 3),
               hard_iron=np.array([_f64(v) for v in base[9:13]]), pivot=float(piv))
    cls = 'regular' if piv > REGULAR else 'band'
    if want_bound or want_cal or model is not None:
        bnd = _bound(pipe, base, seg, mag, t_f, Ns, ext_abs, f)
        out['b_soft'], out['b_hard'] = bnd['y'][0:9].reshape(3, 3), bnd['y'][9:13]
        out['rel'] = bnd['rel']
        if bnd['rel'] > 1e-3:
            cls = 'band'
        if want_cal:
            out['mag_cal'], out['b_cal'] = _mag_cal(mag, seg, base, bnd)
        if model is not None:
            out['err'], out['b_err'] = _err(base, bnd, *model)
    out['cls'] = cls
    return out


def _fsolve(A, b):
    """A^-1 b in Fraction (A nonsingular)."""
    n = len(b)
    M = [list(A[i]) + [b[i]] for i in range(n)]
    for c in range(n):
        p = next(r for r in range(c, n) if M[r][c] != 0)
        M[c], M[p] = M[p], M[c]
        for r in range(n):
            if r != c and M[r][c] != 0:
                f = M[r][c] / M[c][c]
                M[r] = [x - f * y for x, y in zip(M[r], M[c])]
    return [M[i][n] / M[i][i] for i in range(n)]


def _bound(pipe, base, seg, mag, t_f, Ns, ext_abs, f):
    """First-order bound on K10's rounding (module docstring) of y = (S [9], hard [4], O [9], s [3])."""
    P = pipe.last
    mom, t = pipe.mom, pipe.t
    inj = []        # (key, size)
    # the moments: depth of K10's sums, and the term roundings
    for s, (a, b) in enumerate(seg):
        d = np.abs(mag[a:b] - t_f)
        depth = -(-(b - a) // THREADS) + 5 + 7 + 2
        sums = [d[:, i].sum() for i in range(3)] + [(d[:, i] * d[:, j]).sum() for i, j in QUAD] + \
               [(d[:, i] * d[:, j] * d[:, k]).sum() for i, j, k in CUBIC]
        for i, v in enumerate(sums):
            inj.append((('mom', 19 * s + i), gamma(depth + (1 if i < 3 else 3 if i < 9 else 5)) * v * (1 + 1e-12)))
    # the plane solves: formation and elimination errors carried through |A^-1|
    for s in range(3):
        N = Ns[s]
        s1, q = mom[s][0:3], mom[s][3:9]
        Q = _sym3(q)
        A = mp.matrix([[Q[i, j] + t[i] * s1[j] + s1[i] * t[j] + N * t[i] * t[j] for j in range(3)] for i in range(3)])
        dA = mp.matrix([[gamma(5) * (abs(Q[i, j]) + abs(t[i] * s1[j]) + abs(s1[i] * t[j]) + N * abs(t[i] * t[j]))
                         for j in range(3)] for i in range(3)])
        rhs = mp.matrix([s1[i] + N * t[i] for i in range(3)])
        db = mp.matrix([gamma(2) * (abs(s1[i]) + N * abs(t[i])) for i in range(3)])
        x = _solve(A, rhs)
        ax = _absmat(x)
        dx = _absmat(_inv(A)) * (db + (dA + gamma(9) * _lu_abs(A)) * ax)
        nrm = mp.sqrt(sum(v * v for v in x))
        for i in range(3):
            inj.append((('x', 3 * s + i), dx[i]))
            inj.append((('v', 3 * s + i), gamma(5) * abs(x[i]) / nrm))
    # the extremes, the range ratios and S
    for s in range(3):
        for j in range(4):
            inj.append((('ext', 4 * s + j), gamma(3) * ext_abs[s][j // 2] * (1 + 1e-12)))
        inj.append((('r', s), gamma(3)))
    S = P['S']
    for i in range(3):
        for j in range(3):
            inj.append((('Sm', 3 * i + j), gamma(7) * abs(S[i, j])))
    # the sphere solve, equilibrated by f as K10 does: formation and elimination errors
    aS = _absmat(S)
    D1 = mp.matrix([abs(v) for v in P['D'][0:3]])
    D2 = _absmat(_sym3(P['D'][3:9]))
    T3 = _cubic([abs(v) for v in P['D'][9:19]])
    G = aS.T * aS
    aw = mp.matrix([sum(G[b, c] * T3[(a, b, c)] for b in range(3) for c in range(3)) for a in range(3)])
    dU1 = gamma(3) * (aS * D1)
    dU2 = gamma(6) * (aS * D2 * aS.T)
    dv = gamma(15) * (aS * aw)
    f = mp.mpf(f)
    Hf = P['HH'].copy()
    dH = mp.zeros(4, 4)
    for i in range(3):
        for j in range(3):
            Hf[i, j] *= f * f
            dH[i, j] = 4 * dU2[i, j] * f * f
        Hf[i, 3] *= f
        Hf[3, i] *= f
        dH[i, 3] = dH[3, i] = 2 * dU1[i] * f
    pf = mp.matrix([P['p'][0] * f, P['p'][1] * f, P['p'][2] * f, P['p'][3] * f * f])
    dr = mp.matrix([2 * dv[0] * f ** 3, 2 * dv[1] * f ** 3, 2 * dv[2] * f ** 3,
                    (gamma(2) * (abs(P['U2'][0, 0]) + abs(P['U2'][1, 1]) + abs(P['U2'][2, 2])) +
                     dU2[0, 0] + dU2[1, 1] + dU2[2, 2]) * f * f])
    dp = _absmat(_inv(Hf)) * (dr + (dH + gamma(12) * _lu_abs(Hf)) * _absmat(pf))
    for i in range(4):
        inj.append((('q', i), dp[i] / (f if i < 3 else f * f)))
    # first order: each perturbation through the exact pipeline
    b0 = [mp.mpf(0)] * len(base)
    for key, size in inj:
        size = mp.mpf(size)
        if size == 0:
            continue
        y = pipe.run(key=key, val=size * _EPS)
        for k in range(len(base)):
            b0[k] += abs(y[k] - base[k]) / _EPS
    pipe.run()
    # the final roundings: T = S t, hard = q + T, the radius
    p = P['p']
    for i in range(3):
        T = sum(abs(S[i, j] * t[j]) for j in range(3))
        b0[9 + i] += gamma(3) * T + U * (abs(p[i]) + T)
    r = base[12]
    b0[12] += gamma(4) * (abs(p[3]) + p[0] ** 2 + p[1] ** 2 + p[2] ** 2) / (2 * r) + U * r
    for i in range(3):
        b0[22 + i] += gamma(6) * abs(base[22 + i])     # s's own roundings (pass 3 uses s)
    y = np.array([float(SLACK * v) for v in b0])
    scale_S = max(abs(v) for v in base[0:9])
    scale_h = abs(base[12])
    rel = max(max(float(b0[k] / scale_S) for k in range(9)), max(float(b0[k] / scale_h) for k in range(9, 13)))
    return dict(y=y, rel=rel)


def _mag_cal(mag, seg, base, bnd):
    """The staged s_i (O_i m) - hard_i in long double, and its bound from those of O, s, hard and the three
    roundings of the row."""
    ld = np.longdouble
    O = np.array([ld(mp.nstr(v, 30)) for v in base[13:22]], dtype=ld).reshape(3, 3)
    s = np.array([ld(mp.nstr(v, 30)) for v in base[22:25]], dtype=ld)
    h = np.array([ld(mp.nstr(v, 30)) for v in base[9:12]], dtype=ld)
    m = np.concatenate([mag[a:b] for a, b in seg]).astype(ld)
    c = m.dot(O.T)
    cal = s * c - h
    bO, bs, bh = bnd['y'][13:22].reshape(3, 3), bnd['y'][22:25], bnd['y'][9:12]
    am = np.abs(m.astype(np.float64))
    ac = am.dot(np.abs(O.astype(np.float64)).T)
    sf, hf = np.abs(s.astype(np.float64)), np.abs(h.astype(np.float64))
    b = SLACK * (np.abs(c.astype(np.float64)) * bs + sf * am.dot(bO.T) + bh) + gamma(5) * (sf * ac + hf) + \
        2.0 ** -62 * (sf * ac + hf)
    return cal, b


def _err(base, bnd, si, hi, bmag):
    """The generated form's err [13] from the exact S and hard iron, and its bound from theirs: with
    P = S si, k = trace(P) / 3: E = P / k - I, hard[0:3] / k - hi, hard[3] / k - b."""
    si = mp.matrix(np.asarray(si, dtype=np.float64).tolist())
    S = mp.matrix([[base[3 * i + j] for j in range(3)] for i in range(3)])
    h = base[9:13]
    P = S * si
    k = (P[0, 0] + P[1, 1] + P[2, 2]) / 3
    b = mp.mpf(float(bmag))
    e = [P[i, j] / k - (1 if i == j else 0) for i in range(3) for j in range(3)] + \
        [h[i] / k - mp.mpf(float(hi[i])) for i in range(3)] + [h[3] / k - b]
    bS = mp.matrix(bnd['y'][0:9].reshape(3, 3).tolist())
    asi = _absmat(si)
    aP = _absmat(S) * asi
    dP = bS * asi + gamma(3) * aP
    ak = abs(k)
    dk = (dP[0, 0] + dP[1, 1] + dP[2, 2]) / 3 + gamma(4) * (aP[0, 0] + aP[1, 1] + aP[2, 2]) / 3
    be = [SLACK * (dP[i, j] / ak + abs(P[i, j]) * dk / ak ** 2) + gamma(2) * (abs(P[i, j]) / ak + (i == j))
          for i in range(3) for j in range(3)]
    bh = list(bnd['y'][9:13])
    be += [SLACK * (bh[i] / ak + abs(h[i]) * dk / ak ** 2) + gamma(2) * (abs(h[i]) / ak + abs(float(hi[i])))
           for i in range(3)]
    be += [SLACK * (bh[3] / ak + abs(h[3]) * dk / ak ** 2) + gamma(2) * (abs(h[3]) / ak + b)]
    return np.array([_f64(v) for v in e]), np.array([float(v) for v in be])


# ---- the reference's own steps at 200 bits, for checking calibrate --------------------------------------------
def direct_mp(mag, segments, prec=200):
    """calibrate_direct's steps (plane fits on m, staged corrections, ranges over every sample, the [2c, 1]
    sphere fit on c = S m) in mpmath at prec bits: (S [3, 3] mp, hard [4] mp)."""
    with mp.workprec(prec):
        seg = check_segments(segments, np.asarray(mag).shape[0])
        segs = [[[mp.mpf(float(v)) for v in row] for row in np.asarray(mag)[a:b]] for a, b in seg]
        O = []
        for m in segs:
            A = mp.matrix([[sum(r[i] * r[j] for r in m) for j in range(3)] for i in range(3)])
            x = _solve(A, mp.matrix([sum(r[i] for r in m) for i in range(3)]))
            im = max(range(3), key=lambda i: abs(x[i]))
            sg = -1 if x[im] < 0 else 1
            nrm = mp.sqrt(sum(x[i] ** 2 for i in range(3)))
            O.append([sg * x[i] / nrm for i in range(3)])
        cs = [[[sum(O[k][i] * r[i] for i in range(3)) for k in range(3)] for r in m] for m in segs]
        rng = []
        for s, c in enumerate(cs):
            a, b = _RANGE_COLS[s]
            rng.append((max(r[a] for r in c) - min(r[a] for r in c), max(r[b] for r in c) - min(r[b] for r in c)))
        sZ2Y, sZ2X, sY2X = rng[0][0] / rng[0][1], rng[1][0] / rng[1][1], rng[2][0] / rng[2][1]
        sv = [mp.mpf(1), 1 / sY2X, (1 + sY2X * sY2X) / (sY2X * sY2X * sZ2X + sY2X * sZ2Y)]
        c = [[sv[k] * r[k] for k in range(3)] for cc in cs for r in cc]
        H = mp.matrix([[2 * r[0], 2 * r[1], 2 * r[2], 1] for r in c])
        y = mp.matrix([r[0] ** 2 + r[1] ** 2 + r[2] ** 2 for r in c])
        p = _solve(H.T * H, H.T * y)
        S = [[sv[i] * O[i][j] for j in range(3)] for i in range(3)]
        return S, [p[0], p[1], p[2], mp.sqrt(p[3] + p[0] ** 2 + p[1] ** 2 + p[2] ** 2)]
