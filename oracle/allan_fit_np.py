"""IEEE Std 952-1997 Annex C noise identification from an Allan variance curve, in NumPy float64 -- the oracle
of K13 (csrc/allanfit_kernel.cuh).

On the Allan tau grid of n samples at fs (oracle_np.allan_multipliers: m_k = j*10^i <= n/9, tau_k = m_k / fs),
with the weights w_k = floor(n / m_k) - 1 (the number of squared differences allan.allan_var averages at m_k):

    model(tau) = C_-2 tau^-2 + C_-1 tau^-1 + C_0 + C_1 tau + C_2 tau^2,   every C_p >= 0,
    minimise   sum_k w_k (model(tau_k) / v_k - 1)^2              (v_k the variance at tau_k)

over the bins with v_k > 0.  The columns a_kp = sqrt(w_k) tau_k^p / v_k are scaled to unit norm once; the
non-negative least-squares optimum is found by enumerating the 31 non-empty supports S of {-2..2} (bit i of a
support is the term tau^(i-2)): the unconstrained least-squares solution on S (np.linalg.lstsq) is feasible when
every coefficient on S is > 0, and the answer is the feasible support of smallest objective.  The empty support
(objective sum_k w_k) is always feasible.  Supports are visited with fewer terms first, then by bitmask, and a later
one replaces the best only if its objective is lower by more than TIE * sum_k w_k: objectives closer than that are a
tie, and ties go to fewer terms, then to the lower bitmask.  A support is skipped when it has more columns than
usable bins, or when its R factor has a diagonal entry <= RANK * max |diag|.

Outputs (in order): Q = sqrt(C_-2 / 3), N = sqrt(C_-1), B = sqrt(C_0 pi / (2 ln 2)), K = sqrt(3 C_1),
R = sqrt(2 C_2), B_min = sqrt(min_k v_k) / sqrt(2 ln 2 / pi).

Edges: any NaN, +-inf or negative v_k, or an empty grid, gives six NaNs; a bin with v_k = 0 is left out of the fit
but counts for B_min; if every bin is zero the output is all zeros."""
import numpy as np

from oracle_np import allan_multipliers

TIE = 1e-12
RANK = 1e-13
# evaluation order: fewer terms first, then the lower bitmask
SUPPORTS = sorted(range(1, 32), key=lambda s: (bin(s).count('1'), s))
B_SCALE = np.sqrt(np.pi / (2.0 * np.log(2.0)))      # B = sqrt(C_0) * B_SCALE; B_min = min dev * B_SCALE


def grid(n, fs):
    """(tau [ntau], w [ntau]) of the Allan grid of n samples at fs; tau as allan.py:58 forms it."""
    mult = np.asarray(allan_multipliers(n, fs), dtype=np.int64)
    return mult.astype(np.float64) * (1.0 / float(fs)), (n // mult - 1).astype(np.float64)


def outputs(C, vmin):
    """The six outputs from the coefficients C [5] (C_-2 .. C_2) and the smallest variance."""
    C = np.asarray(C, dtype=np.float64)
    return np.array([np.sqrt(C[0] / 3.0), np.sqrt(C[1]), np.sqrt(C[2]) * B_SCALE, np.sqrt(3.0 * C[3]),
                     np.sqrt(2.0 * C[4]), np.sqrt(vmin) * B_SCALE])


def system(v, tau, w):
    """The scaled system of the usable bins: D [U, 5] (unit columns), b [U], the column norms s [5] and the
    usable mask."""
    use = v > 0.0
    p = np.arange(-2, 3)
    A = np.sqrt(w[use])[:, None] * tau[use][:, None] ** p[None, :] / v[use][:, None]
    s = np.linalg.norm(A, axis=0)
    return A / s, np.sqrt(w[use]), s, use


def solve_support(D, b, mask):
    """(y [5] with zeros off the support, objective) of the unconstrained fit on support `mask`, or None when the
    support is skipped (more columns than rows, or a rank-deficient R)."""
    cols = [i for i in range(5) if mask >> i & 1]
    if len(cols) > D.shape[0]:
        return None
    Ds = D[:, cols]
    d = np.abs(np.diag(np.linalg.qr(Ds, mode='r')))
    if not np.all(d > RANK * d.max()):
        return None
    ys = np.linalg.lstsq(Ds, b, rcond=None)[0]
    y = np.zeros(5)
    y[cols] = ys
    r = Ds @ ys - b
    return y, float(np.sum(r * r))


def fit(v, n, fs, detail=False):
    """Six outputs of one variance curve v [ntau] on the grid of (n, fs).  detail: also a dict with the chosen
    support 'mask' (0: empty), the coefficients 'C' [5], its 'objective', 'W' = sum w, 'objectives' {mask: objective}
    of every feasible support (empty included) and 'runner_up', the smallest objective of the others."""
    v = np.asarray(v, dtype=np.float64)
    tau, w = grid(n, fs)
    if v.shape != tau.shape:
        raise ValueError('the curve has %d bins, the grid of n=%d at fs=%g has %d' % (v.size, n, fs, tau.size))
    info = {'mask': None, 'C': np.full(5, np.nan), 'objective': np.nan, 'W': np.nan, 'objectives': {},
            'runner_up': np.nan}
    if v.size == 0 or not np.all(np.isfinite(v)) or np.any(v < 0.0):
        out = np.full(6, np.nan)
        return (out, info) if detail else out
    D, b, s, use = system(v, tau, w)
    W = float(np.sum(w[use]))
    best_mask, best_y, best_obj = 0, np.zeros(5), W
    objs = {0: W}
    if use.any():
        for mask in SUPPORTS:
            got = solve_support(D, b, mask)
            if got is None:
                continue
            y, obj = got
            if not np.all(y[[i for i in range(5) if mask >> i & 1]] > 0.0):
                continue
            objs[mask] = obj
            if obj < best_obj - TIE * W:
                best_mask, best_y, best_obj = mask, y, obj
    C = np.where(best_y != 0.0, best_y / np.where(s > 0.0, s, 1.0), 0.0) if use.any() else np.zeros(5)
    out = outputs(C, v.min())
    if detail:
        others = [o for m, o in objs.items() if m != best_mask]
        info = {'mask': best_mask, 'C': C, 'objective': best_obj, 'W': W, 'objectives': objs,
                'runner_up': min(others) if others else np.inf}
        return out, info
    return out


def fit_batch(var, n, fs):
    """[nseries, 6] outputs of var [nseries, ntau]."""
    var = np.asarray(var, dtype=np.float64)
    return np.stack([fit(v, n, fs) for v in var.reshape(-1, var.shape[-1])]) if var.size else \
        np.full((int(np.prod(var.shape[:-1])), 6), np.nan)


def model_curve(C, n, fs):
    """sigma^2(tau_k) of the coefficients C [5] on the grid of (n, fs)."""
    tau, _ = grid(n, fs)
    return sum(C[i] * tau ** (i - 2) for i in range(5))


# ---- laws: what the fit returns on noise of known coefficients (1 h at 100 Hz) ----------------------------------
# Each case: the output column, the true value, and the oracle's ratio estimate / truth over NumPy-generated series
# (mean, standard deviation over series) with a per-series envelope.  The relative weighting biases the long-tau
# terms (K, R) low; these are the oracle's numbers, not an unbiased target.  The CPU tests regenerate them
# (tests/test_cpu_allan_fit.py); the GPU tests hold the device path, through Sim and logged directories, to them.
LAW_FS, LAW_N = 100.0, 360000
LAWS = {
    # white rate noise, N = arw
    'white': dict(col=1, truth=1e-3, mean=0.9995, sd=0.0016, lo=0.99, hi=1.01),
    # white (N = 1e-4) plus a random walk of the rate, K = 3e-5
    'rw': dict(col=3, truth=3e-5, mean=0.945, sd=0.067, lo=0.6, hi=1.3),
    # white (N = 1e-3) plus a rate ramp, R = 1e-6
    'ramp': dict(col=4, truth=1e-6, mean=0.90, sd=0.10, lo=0.45, hi=1.35),
    # white angle increments (N = 1e-4) of an angle quantised to q = 1e-5, differenced: Q = q / sqrt(12)
    'quant': dict(col=0, truth=1e-5 / np.sqrt(12.0), mean=1.006, sd=0.019, lo=0.9, hi=1.1),
}


def law_series(kind, rng, fs=LAW_FS, n=LAW_N):
    """One NumPy-generated rate series [n] of law case `kind`."""
    dt = 1.0 / fs
    if kind == 'white':
        return 1e-3 * np.sqrt(fs) * rng.standard_normal(n)
    if kind == 'rw':
        return 1e-4 * np.sqrt(fs) * rng.standard_normal(n) + np.cumsum(3e-5 * np.sqrt(dt) * rng.standard_normal(n))
    if kind == 'ramp':
        return 1e-3 * np.sqrt(fs) * rng.standard_normal(n) + 1e-6 * np.arange(n) * dt
    if kind == 'quant':
        q = 1e-5
        th = np.concatenate([[0.0], np.cumsum(1e-4 * np.sqrt(fs) * rng.standard_normal(n) * dt)])
        return np.diff(q * np.floor(th / q + 0.5)) / dt
    raise ValueError(kind)


def law_check(kind, ratios):
    """Every ratio inside the case's envelope, and their mean within 5 standard errors of the oracle's mean."""
    c = LAWS[kind]
    r = np.asarray(ratios, dtype=np.float64).reshape(-1)
    inside = bool(np.all((r >= c['lo']) & (r <= c['hi'])))
    mean_ok = abs(r.mean() - c['mean']) <= 5.0 * c['sd'] / np.sqrt(r.size)
    return inside and mean_ok, (r.min(), r.mean(), r.max())
