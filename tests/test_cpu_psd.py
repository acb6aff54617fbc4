"""K5's plan table and the reference the PSD tests lean on, without a GPU.

b2ins_diag_psd_plan reports which transform b2ins_psd_series_f64 takes for a length (the direct cosine
synthesis, radix-2 or Bluestein); tests/test_gpu_psd.py picks its lengths to reach every plan and its edges,
and this file keeps those claims true.  oracle/psd_exact.py evaluates the same cosine synthesis as
time_series_from_psd with exactly reduced angles and wide sums; it certifies the float64 oracle the GPU tests
compare K5 with."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT, load_golden
import oracle_np as onp
import psd_exact

# n -> (plan, transform length) for every length tests/test_gpu_psd.py sweeps, and the plan boundaries
PLANS = {
    1: ('direct', 0), 2: ('direct', 0), 3: ('direct', 0), 5: ('direct', 0),
    13: ('direct', 0), 14: ('direct', 0),                                  # M = 7: the largest direct M below 8
    15: ('radix2', 8), 16: ('radix2', 8), 32: ('radix2', 16), 64: ('radix2', 32),
    18: ('bluestein', 32), 34: ('bluestein', 64), 1000: ('bluestein', 1024), 777: ('bluestein', 1024),
    2050: ('bluestein', 4096),
    4098: ('bluestein', 8192),                                             # M = 2049: the first M with P = 8192
    8186: ('bluestein', 8192),                                             # M = 4093, prime
    8190: ('bluestein', 8192),                                             # M = 4095: the last Bluestein M
    8192: ('radix2', 4096),                                                # M = 4096
    8193: ('direct', 0), 8194: ('direct', 0),                              # M = 4097: the first direct M above
    10000: ('direct', 0),
    16382: ('direct', 0),                                                  # M = 8191, prime
    16383: ('radix2', 8192), 16384: ('radix2', 8192), 16385: ('radix2', 8192), 40001: ('radix2', 8192),
}
FS = 200.0


def _is_prime(m):
    return m > 1 and all(m % d for d in range(2, math.isqrt(m) + 1))


def _plan_env():
    if os.environ.get('B2INS_PSD_DIRECT') is not None:
        pytest.skip('B2INS_PSD_DIRECT is set in this process: every length takes the direct synthesis')
    from gnss_ins_sim_b200 import _lib
    return _lib


def test_plan_of_every_swept_length():
    _lib = _plan_env()
    for n, want in sorted(PLANS.items()):
        assert _lib.psd_plan(n) == want, (n, _lib.psd_plan(n), want)
    assert _is_prime(4093) and _is_prime(8191)


def test_plan_follows_the_series_length_rule():
    """Every n up to 40001: N = n rounded up to even, at most 16384, M = N / 2; radix-2 of length M for a
    power-of-two M >= 8, Bluestein of length 2^ceil(log2(2M - 1)) <= 8192 for the other M in 9 .. 4095, the
    direct synthesis otherwise."""
    _lib = _plan_env()
    lib = _lib.load()
    seen = set()
    for n in range(1, 40002):
        N = min(n + n % 2, 16384)
        assert lib.b2ins_psd_series_len(n) == N
        M = N // 2
        if M >= 8 and M & (M - 1) == 0:
            want = ('radix2', M)
        elif 9 <= M <= 4095:
            want = ('bluestein', 1 << (2 * M - 2).bit_length())
        else:
            want = ('direct', 0)
        if n in PLANS or n % 97 == 0 or M in (7, 8, 9, 4095, 4096, 4097, 8191, 8192):
            got = _lib.psd_plan(n)
            assert got == want, (n, got, want)
            seen.add(got[0])
        assert want[1] <= 8192
    assert seen == {'direct', 'radix2', 'bluestein'}
    with pytest.raises(ValueError):
        _lib.psd_plan(0)


def test_direct_override_is_reported():
    """With B2INS_PSD_DIRECT set (latched once per process) every length reports the direct synthesis."""
    code = ('import sys; sys.path.insert(0, %r)\n'
            'from gnss_ins_sim_b200 import _lib\n'
            'print(sorted({_lib.psd_plan(n) for n in (16, 1000, 8190, 16384, 40001)}))\n') % ROOT
    env = dict(os.environ, B2INS_PSD_DIRECT='1')
    out = subprocess.run([sys.executable, '-c', code], env=env, cwd=ROOT, capture_output=True, text=True,
                         timeout=120)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "[('direct', 0)]", out.stdout


def test_exact_synthesis_of_single_bins():
    """One bin at a time: the synthesis is (2/N) (A cos - B sin)(2 pi k m / N), (A_0 / N) or ((-1)^m A_M / N)."""
    for N in (2, 6, 14, 18, 1000):
        L = N // 2 + 1
        m = np.arange(N)
        for k in sorted({0, 1, L // 2, L - 2, L - 1}):
            A, B = np.zeros(L), np.zeros(L)
            A[k], B[k] = 0.75, -1.25
            x = psd_exact.cosine_synthesis(A, B, N)
            if k == 0:
                ref = np.full(N, 0.75 / N)
            elif k == L - 1:
                ref = np.where(m % 2 == 0, 0.75, -0.75) / N
            else:
                th = [2.0 * math.pi * ((k * mm) % N) / N for mm in m]
                ref = np.array([2.0 * (0.75 * math.cos(t) + 1.25 * math.sin(t)) / N for t in th])
            assert np.abs(x - ref).max() <= 1e-14 * np.abs(ref).max(), (N, k, np.abs(x - ref).max())


@pytest.mark.parametrize('n', [1, 2, 3, 5, 14, 16, 18, 32, 34, 777, 1000, 2050, 4098, 8186, 8190, 8192, 8193])
def test_oracle_transform_is_exact_to_1e_14(n):
    """time_series_from_psd (np.fft) against the exact synthesis of the same bins, on the golden table
    (interpolated to every length), at <= 1e-14 of the series maximum, for one run per sensor and axis."""
    g = load_golden('psd.npz')
    freq, sxx = g['freq_a'], g['sxx_a']
    fs = float(g['fs_a'])
    tabs = (sxx, 2.0 * sxx, 0.5 * sxx + 1e-6)
    N = min(n + n % 2, 16384)
    worst = 0.0
    for sensor in (0, 1):
        z = onp.psd_phase_normals(N // 2 + 1, [7], 99, sensor)[0]
        for c in range(3 if N < 4096 else 1):
            ok, x = onp.time_series_from_psd(tabs[c], freq, fs, n, z[c])
            ok2, xe = psd_exact.time_series_from_psd(tabs[c], freq, fs, n, z[c])
            assert ok and ok2 and x.shape == xe.shape == (n,)
            scale = np.abs(xe).max()
            assert scale > 0.0
            worst = max(worst, np.abs(x - xe).max() / scale)
    print('n = %d: time_series_from_psd vs exact synthesis, worst %.2e of max|x|' % (n, worst))
    assert worst <= 1e-14, (n, worst)
