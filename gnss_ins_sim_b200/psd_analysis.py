"""Psd plugin -- Welch power spectral density of the accelerometer and gyroscope channels
(input ['fs','accel','gyro'], output ['algo_freq','psd_accel','psd_gyro']), with the semantics of
scipy.signal.welch; the estimator itself is csrc/welch_kernel.cuh (K11)."""
import numpy as np

from . import engine
from .series_analysis import SeriesEstimator


class Psd(SeriesEstimator):
    '''
    One-sided power spectral density of the three accelerometer and three gyroscope channels by Welch's
    method, as scipy.signal.welch(x, fs, window, nperseg, noverlap) computes it (detrend='constant',
    scaling='density', average='mean', nfft = nperseg): segments of nperseg samples, noverlap of them shared
    with the next (default nperseg // 2), each with its mean removed and windowed; the squared magnitudes of
    their transforms are averaged.  Units: (m/s^2)^2/Hz and (rad/s)^2/Hz.  A white noise of density
    sigma / sqrt(Hz) gives a floor of 2 sigma^2.

    nperseg: even, >= 16, and a power of two up to 16384 or at most 8192.
    window: 'hann' (scipy's periodic Hann, 0.5 - 0.5 cos(2 pi m / nperseg)) or any finite array of nperseg
    values (np.ones(nperseg) is the boxcar window).
    '''

    def __init__(self, nperseg=256, noverlap=None, window='hann'):
        if isinstance(nperseg, (bool, np.bool_)) or not isinstance(nperseg, (int, np.integer)):
            raise TypeError('nperseg must be an int, got %r' % (nperseg,))
        self.nperseg = N = int(nperseg)
        if engine.welch_workspace_bytes(N, 1, N, 0) < 0:
            raise ValueError('nperseg=%d: need an even length >= 16, a power of two up to 16384 or at most 8192'
                             % N)
        if noverlap is None:
            noverlap = N // 2
        if isinstance(noverlap, (bool, np.bool_)) or not isinstance(noverlap, (int, np.integer)):
            raise TypeError('noverlap must be an int or None, got %r' % (noverlap,))
        if not 0 <= noverlap < N:
            raise ValueError('need 0 <= noverlap < nperseg, got noverlap=%d, nperseg=%d' % (noverlap, N))
        self.noverlap = int(noverlap)
        if isinstance(window, str):
            if window != 'hann':
                raise ValueError("window must be 'hann' or an array of nperseg values, got %r" % (window,))
            w = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(N) / N)
        else:
            try:
                w = np.array(window, dtype=np.float64)
            except (TypeError, ValueError):
                raise TypeError('window must be \'hann\' or an array of nperseg values, got %r' % (window,))
            if w.shape != (N,):
                raise ValueError('window must have shape (%d,), got %s' % (N, w.shape))
            if not np.all(np.isfinite(w)):
                raise ValueError('window values must be finite')
        self.window = w
        super().__init__(['algo_freq', 'psd_accel', 'psd_gyro'])

    def _series(self, fs, x, n, nseries, **addressing):
        if n < self.nperseg:
            raise ValueError('a series of %d samples is shorter than nperseg=%d' % (n, self.nperseg))
        return engine.welch(fs, x, n, nseries, self.nperseg, self.noverlap, self.window, **addressing)

    def frequencies(self, fs):
        '''freq [L] of run_batch for sample rate fs: k / (nperseg (1/fs)), as np.fft.rfftfreq.'''
        return np.arange(self.nperseg // 2 + 1) * (1.0 / (self.nperseg * (1.0 / fs)))

    def abscissa(self, n, fs):
        return self.frequencies(fs)

    def run_bytes(self, n):
        # K1's 48 B per run-sample, then K11's chunk sums for the six series of a run
        return 48 + max(engine.welch_workspace_bytes(n, 6, self.nperseg, self.noverlap), 0) / n
