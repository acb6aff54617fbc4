"""The exact Gauss-Markov drift (oracle/gm_exact.py) and K1's noise plan (b2ins_diag_noise_plan), without a GPU.

gm_exact is held to a Fraction evaluation of d_t = sum_{k<t} a^(t-1-k) b z_k on short series, for every class
of decay factor a the generators meet, and bounds the serial float64 recurrence of the reference
(oracle_np.bias_drift: a product and a sum per step) by 2 u Psi_t.  The plan is the host function the K1 / K9
launch calls: its coefficients are the reference's, and pass 1 of the segmented path only drops drives whose
weight at the segment end, |a|^pass1_len, is below 1e-20 for every channel."""
import math
from fractions import Fraction

import numpy as np
import pytest

import gm_exact as ge
import oracle_np as onp

U = 2.0 ** -53
FS = 100.0
DT = 1.0 / FS

# correlation times against dt = 0.01 s, by the class of a = 1 - dt / tau they give
TAUS = {'tau=100s': 100.0, 'near random walk': 1e7, 'tau=3dt': 3 * DT, 'a=0': DT, 'a=-1/3': 0.75 * DT,
        'a=-0.99': DT / 1.99, 'a=-1': DT / 2}


def _err(corr, drift, white_key):
    c = np.broadcast_to(np.asarray(corr, dtype=np.float64), (3,)).copy()
    d = np.broadcast_to(np.asarray(drift, dtype=np.float64), (3,)).copy()
    return {'b': np.zeros(3), 'b_drift': d, 'b_corr': c, white_key: np.zeros(3)}


def _plan(gyro_corr, accel_corr, runs=3, n=300001, sms=132):
    from gnss_ins_sim_b200 import _lib
    return _lib.noise_plan(FS, runs, n, _err(gyro_corr, 1e-5, 'arw'), _err(accel_corr, 1e-3, 'vrw'), sms)


def _fraction_drift(a, b, z):
    A, B = Fraction(float(a)), Fraction(float(b))
    D, out = Fraction(0), [0.0]
    for k in range(len(z) - 1):
        D = A * D + B * Fraction(float(z[k]))
        out.append(float(D))
    return np.array(out)


@pytest.mark.parametrize('a', [0.9999, 1.0 - 1e-9, 2.0 / 3.0, 0.0, -1.0 / 3.0, -0.99, -1.0, 1.0, -3.0, 1.5])
def test_exact_drift_equals_fractions(a):
    rng = np.random.default_rng(7)
    z = rng.standard_normal(61)
    z[5] = 0.0
    z[9] = 2.0 ** -1070                      # a subnormal drive
    for b in (1.7e-5, 3.0, 2.0 ** -600, 0.0):
        d, psi = ge.drift(a, b, z)
        assert np.array_equal(d, _fraction_drift(a, b, z)), (a, b)
        assert np.all(psi >= np.abs(d)) and psi[0] == 0.0


@pytest.mark.parametrize('name', list(TAUS))
def test_reference_recurrence_within_the_serial_bound(name):
    """oracle_np.bias_drift: d_{t+1} = fl(fl(a d_t) + fl(b z_t)), two roundings and the drive's product per
    step, so |d - exact| <= 2 u Psi_t (first order; Psi_t >= |d_t| holds the rounding of the exact value)."""
    tau = TAUS[name]
    n, R = 4000, 2
    z = np.random.default_rng(3).standard_normal((R, n, 3))
    corr = np.array([tau, tau, np.inf])
    drift_ = np.array([1e-5, 2.0, 1e-5])
    ref = onp.bias_drift(corr, drift_, n, FS, z)
    a, b = onp.gm_coeffs(corr, drift_, FS)
    worst = 0.0
    for c in range(2):
        d, psi = ge.drift(np.full(R, a[c]), np.full(R, b[c]), z[:, :, c])
        bound = (2 * U * psi) * (1 + 4 * n * U) + U * np.abs(d)
        err = np.abs(ref[:, :, c] - d)
        assert np.all(err <= bound), (name, c, np.max(err / np.where(bound > 0, bound, 1)))
        worst = max(worst, float(np.max(err / np.where(bound > 0, bound, np.inf))))
    # the white channel is drift * z, one product: exactly the generators' fl(wd z)
    assert np.array_equal(ref[:, :, 2], drift_[2] * z[:, :, 2])
    assert worst < 1.0


def test_digested_coefficients_are_the_reference_ones():
    """gm_a is 1 - 1/fs/tau exactly as pathgen.py:583 writes it, bit for bit; gm_b = drift sqrt(1 - exp(-2/(fs
    tau))) (:586) is the same expression through the C library's exp and sqrt; a white channel has gm_a = gm_b
    = 0 and wd = drift.  The GPU tests take the coefficients from the plan, so an ulp of exp between libraries
    does not enter their bounds."""
    taus = np.array(list(TAUS.values()))
    for i in range(0, len(taus), 3):
        g = np.concatenate([taus[i:i + 3], np.full(3, np.inf)])[:3]
        acc = np.array([taus[(i + 3) % len(taus)], np.inf, 50.0])
        p = _plan(g, acc)
        for corr, drift_, sl in ((acc, 1e-3, slice(0, 3)), (g, 1e-5, slice(3, 6))):
            a, b = onp.gm_coeffs(corr, np.full(3, drift_), FS)
            fin = np.isfinite(corr)
            assert np.array_equal(p['gm_a'][sl][fin], a[fin]), corr
            # gm_b: the host's libm (math.exp / math.sqrt) bit for bit; NumPy's vectorised exp may differ from
            # it by an ulp, which 1 - exp(-2 dt / tau) magnifies by exp / (1 - exp) for long tau (3e-8 at 1e7 s)
            bm = np.array([drift_ * math.sqrt(1.0 - math.exp(-2 / (FS * t))) if np.isfinite(t) else 0.0
                           for t in corr])
            assert np.array_equal(p['gm_b'][sl][fin], bm[fin]), corr
            e = np.exp(-2 / (FS * corr[fin]))
            amp = np.spacing(e) / (1.0 - e) + 2 * U      # an ulp of exp, through 1 - e and the square root
            assert np.all(np.abs(p['gm_b'][sl][fin] - b[fin]) <= amp * b[fin]), corr
            assert np.all(p['wd'][sl][fin] == 0.0)
            assert np.all(p['gm_a'][sl][~fin] == 0.0) and np.all(p['gm_b'][sl][~fin] == 0.0)
            assert np.all(p['wd'][sl][~fin] == drift_)
    p = _plan([DT / 2, DT, 0.75 * DT], [np.inf] * 3)
    assert p['gm_a'][3] == -1.0 and p['gm_a'][4] == 0.0 and p['gm_a'][5] == 1.0 - 1.0 / FS / (0.75 * DT)


# tau such that |a|^2680 = 1e-10: pass 1 holds 2688 samples if its threshold were 1e-10, 5376 at 1e-20
TAU_2688 = DT / (1.0 - math.exp(math.log(1e-10) / 2680))

MIXES = {
    'tau=100s': ([100.0, np.inf, np.inf], [np.inf] * 3),
    'tau=0.99s': ([TAU_2688, np.inf, np.inf], [np.inf] * 3),
    'near random walk': ([1e7, np.inf, np.inf], [np.inf] * 3),
    'short positive': ([3 * DT, DT, np.inf], [0.5, np.inf, np.inf]),
    'a=-1/3': ([0.75 * DT, np.inf, np.inf], [np.inf] * 3),
    'a=-0.99': ([DT / 1.99, np.inf, np.inf], [np.inf] * 3),
    'a=-1': ([DT / 2, np.inf, np.inf], [np.inf] * 3),
    'a=-1 among short ones': ([DT / 2, 3 * DT, DT], [0.75 * DT, 0.01, np.inf]),
    'a=-0.99 in the accel': ([np.inf] * 3, [np.inf, DT / 1.99, 3 * DT]),
    'all white': ([np.inf] * 3, [np.inf] * 3),
}


@pytest.mark.parametrize('mix', list(MIXES))
@pytest.mark.parametrize('runs,n', [(3, 300001), (1, 1 << 18), (2, 5 * 10 ** 6), (300, 300001)])
def test_pass1_covers_every_drive_that_still_matters(mix, runs, n):
    """For every channel: pass1_len = seg_len, or |a|^pass1_len < 1e-20.  Segments hold whole 896-sample
    tiles and cover the series; pass 1 holds whole tiles too."""
    g, acc = MIXES[mix]
    p = _plan(g, acc, runs=runs, n=n)
    nseg, L, p1 = p['nseg'], p['seg_len'], p['pass1_len']
    if runs >= 264:
        assert nseg == 1 and L == n and p1 == 0
        return
    assert nseg >= 2 and L % 896 == 0 and (nseg - 1) * L < n <= nseg * L
    assert 896 <= p1 <= L and (p1 % 896 == 0 or p1 == L)
    for c in range(6):
        a = abs(p['gm_a'][c])
        assert p1 == L or a ** p1 < 1e-20, (mix, c, p['gm_a'][c], p1, L)
    if mix in ('tau=0.99s', 'a=-0.99'):
        assert p1 == 5376
    if mix in ('tau=100s', 'near random walk', 'a=-1', 'a=-1 among short ones'):
        assert p1 == L


def test_plan_segments_against_the_sm_count():
    """No segments for 2 sms runs or more, or below 2^18 samples; otherwise about 2 sms CTAs, each segment
    at least 2^16 samples."""
    e = ([100.0] * 3, [100.0] * 3)
    assert _plan(*e, runs=264, n=10 ** 6)['nseg'] == 1
    assert _plan(*e, runs=1, n=(1 << 18) - 1)['nseg'] == 1
    for runs, n, sms, want in ((1, 1 << 24, 132, (254, 66304)), (3, 300001, 132, (4, 75264)),
                               (2, 10 ** 6, 8, (8, 125440)), (3, 300001, 1, (1, 300001))):
        p = _plan(*e, runs=runs, n=n, sms=sms)
        assert (p['nseg'], p['seg_len']) == want, (runs, n, sms)
