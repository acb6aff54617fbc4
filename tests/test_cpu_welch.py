"""Welch power spectral density (K11) without a GPU: the NumPy oracle against scipy.signal.welch over a grid of
lengths, overlaps, ragged series and windows; the non-finite rule; the two identities the GPU tests rest on (a
K5 series is inverted exactly, a sinusoid's power sits in three Hann bins); the plugin's attributes and
constructor errors; and which lengths the C library accepts."""
import numpy as np
import pytest

import oracle_np as onp
import welch_np as wn

signal = pytest.importorskip('scipy.signal')

NS = [16, 256, 1000, 4096, 6000, 16384]


def _overlaps(N):
    return sorted({0, N // 2, N - 1, N // 2 - 3 if (N // 2) % 2 == 0 else N // 2})


def _close(a, b, rel):
    scale = np.abs(b).max()
    assert np.all(np.abs(a - b) <= rel * np.maximum(np.abs(b), scale * 1e-3)), np.abs(a - b).max() / scale


@pytest.mark.parametrize('N', NS)
def test_oracle_matches_scipy_on_the_grid(N):
    rng = np.random.default_rng(N)
    for D in _overlaps(N):
        S = N - D
        for n in (N, N + S - 1, 3 * N + 7):
            x = rng.standard_normal(n) * 0.3 + 5.0
            for window in ('hann', rng.uniform(0.2, 1.0, N)):
                f, p = wn.welch(x, 200.0, N, D, window)
                fr, pr = signal.welch(x, 200.0, window=window, nperseg=N, noverlap=D)
                assert np.array_equal(f, fr)
                _close(p, pr, 1e-12)


@pytest.mark.parametrize('bad', [np.nan, np.inf, -np.inf])
def test_non_finite_rule_matches_scipy(bad):
    N, D = 256, 128
    x = np.random.default_rng(1).standard_normal(1000)
    K, S = wn.segments(x.size, N, D)
    for i in (0, 77, S * (K - 1) + N - 1):       # first sample, inside, last used sample
        y = x.copy()
        y[i] = bad
        _, p = wn.welch(y, 10.0, N, D)
        _, pr = signal.welch(y, 10.0, nperseg=N, noverlap=D)
        assert np.all(np.isnan(p)) and np.all(np.isnan(pr))
    y = x.copy()
    y[S * (K - 1) + N:] = bad                    # the unused tail is never read
    assert S * (K - 1) + N < y.size
    _, p = wn.welch(y, 10.0, N, D)
    _, pr = signal.welch(y, 10.0, nperseg=N, noverlap=D)
    assert np.all(np.isfinite(p))
    _close(p, pr, 1e-12)


@pytest.mark.parametrize('n', [256, 1000, 6000, 16384])
def test_k5_series_is_inverted_exactly(n):
    """A K5 series of even n <= 16384 has period n; one boxcar segment of n samples returns the table at every
    interior bin (bins 0 and L-1 carry random phases that the real part drops)."""
    fs = 100.0
    tf = np.linspace(0.0, fs / 2, 7)
    tab = np.array([1e-4, 3e-3, 5e-4, 2e-3, 1e-5, 4e-4, 1e-4])
    z = onp.psd_phase_normals(n // 2 + 1, [3], 11, 0)[0, 0]
    ok, x = onp.time_series_from_psd(tab, tf, fs, n, z)
    assert ok and x.size == n
    f, p = wn.welch(x, fs, n, None, np.ones(n))
    want = np.interp(f, tf, tab)
    assert np.abs(p[1:-1] / want[1:-1] - 1).max() <= 8e-12


def test_sinusoid_power_in_three_hann_bins():
    fs, N, A = 400.0, 1024, 0.7
    k0 = 100
    t = np.arange(40 * N) / fs
    x = A * np.sin(2 * np.pi * (k0 * fs / N) * t)
    f, p = wn.welch(x, fs, N)
    assert abs(p[k0 - 1:k0 + 2].sum() * fs / N - A * A / 2) <= 2e-15 * 8
    fr, pr = signal.welch(x, fs, nperseg=N)
    assert abs(pr[k0 - 1:k0 + 2].sum() * fs / N - A * A / 2) <= 2e-15 * 8


def test_white_noise_floor_is_twice_the_variance_over_fs():
    fs, sigma = 100.0, 0.01
    x = np.random.default_rng(5).standard_normal(2 ** 20) * sigma
    _, p = wn.welch(x, fs, 512)
    assert abs(p[1:-1].mean() / (2 * sigma ** 2 / fs) - 1) < 0.01


# ---- plugin and C library (the library loads without a device) ------------------------------------------
@pytest.fixture(scope='module')
def Psd():
    pytest.importorskip('torch')
    from gnss_ins_sim_b200.psd_analysis import Psd
    return Psd


def test_plugin_attributes(Psd):
    p = Psd()
    assert p.input == ['fs', 'accel', 'gyro'] and p.output == ['algo_freq', 'psd_accel', 'psd_gyro']
    assert p.batch is True and p.get_results() is None
    assert p.nperseg == 256 and p.noverlap == 128
    assert np.abs(p.window - signal.get_window('hann', 256)).max() <= 4e-16
    q = Psd(nperseg=6000, noverlap=17, window=np.ones(6000))
    assert q.noverlap == 17 and np.array_equal(q.window, np.ones(6000))
    assert np.array_equal(q.frequencies(400.0), np.fft.rfftfreq(6000, 1 / 400.0))
    p.reset()


@pytest.mark.parametrize('kw, err', [
    (dict(nperseg=255), ValueError), (dict(nperseg=8), ValueError), (dict(nperseg=32768), ValueError),
    (dict(nperseg=8194), ValueError), (dict(nperseg=256.0), TypeError), (dict(nperseg=True), TypeError),
    (dict(noverlap=256), ValueError), (dict(noverlap=-1), ValueError), (dict(noverlap=1.5), TypeError),
    (dict(window='hamming'), ValueError), (dict(window=np.ones(255)), ValueError),
    (dict(window=np.ones((2, 128))), ValueError), (dict(window=np.r_[np.ones(255), np.nan]), ValueError),
    (dict(window=object()), TypeError),
])
def test_plugin_constructor_errors(Psd, kw, err):
    with pytest.raises(err):
        Psd(**kw)


def test_plugin_does_not_import_the_oracle():
    import gnss_ins_sim_b200.psd_analysis as mod
    src = open(mod.__file__).read()
    assert 'oracle' not in src.split('"""', 2)[2]


def test_workspace_bytes_accepts_exactly_the_valid_lengths():
    pytest.importorskip('torch')
    from gnss_ins_sim_b200 import engine
    valid = set()
    for N in range(0, 16385 + 2):
        if engine.welch_workspace_bytes(N, 1, N, 0) >= 0:
            valid.add(N)
    pow2 = {2 ** k for k in range(4, 15)}
    want = {N for N in range(16, 8193, 2)} | pow2
    assert valid == want
    assert engine.welch_workspace_bytes(1000, 1, 256, 256) < 0       # noverlap = nperseg
    assert engine.welch_workspace_bytes(1000, 1, 256, -1) < 0
    assert engine.welch_workspace_bytes(255, 1, 256, 128) < 0        # n < nperseg
    assert engine.welch_workspace_bytes(1000, 7, 256, 128) >= 16
