"""Welch power spectral density restated in NumPy (np.fft.rfft): scipy.signal.welch(x, fs, window, nperseg,
noverlap) with detrend='constant', scaling='density', average='mean', one-sided, nfft = nperseg.

    N = nperseg, D = noverlap, S = N - D, K = (n - D) // S segments (samples after the last are unused)
    y_j[m] = (x[jS + m] - mean_m x[jS + m]) w[m]
    psd[k] = (1/K) sum_j c_k |rfft(y_j)[k]|^2 / (fs sum w^2),  c_0 = c_{L-1} = 1, else 2,  L = N/2 + 1
    freq = np.fft.rfftfreq(N, 1/fs)

Non-finite samples: a NaN or +-inf inside a used segment makes every bin NaN (the mean removal spreads it over
the segment, and the transform over every bin); a non-finite sample past the last segment is never read.
This module applies that rule explicitly rather than relying on what the arithmetic happens to give."""
import numpy as np


def hann(N):
    """scipy's periodic Hann window, w[m] = 0.5 - 0.5 cos(2 pi m / N)."""
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(N) / N)


def segments(n, nperseg, noverlap):
    """Number of segments K and the step S."""
    S = nperseg - noverlap
    return (n - noverlap) // S, S


def welch(x, fs, nperseg, noverlap=None, window='hann'):
    """(freq [L], psd [L]) of one series x [n]."""
    x = np.asarray(x, dtype=np.float64)
    N = int(nperseg)
    D = N // 2 if noverlap is None else int(noverlap)
    if not (N % 2 == 0 and 0 <= D < N and x.size >= N):
        raise ValueError('need even nperseg <= n and 0 <= noverlap < nperseg')
    w = hann(N) if isinstance(window, str) else np.asarray(window, dtype=np.float64)
    K, S = segments(x.size, N, D)
    L = N // 2 + 1
    freq = np.fft.rfftfreq(N, 1.0 / fs)
    segs = np.lib.stride_tricks.sliding_window_view(x, N)[::S][:K]
    if not np.all(np.isfinite(segs)):
        return freq, np.full(L, np.nan)
    y = (segs - segs.mean(axis=1, keepdims=True)) * w
    p = np.abs(np.fft.rfft(y, axis=1)) ** 2 / (fs * np.sum(w * w))
    p[:, 1:L - 1] *= 2.0
    return freq, p.mean(axis=0)
