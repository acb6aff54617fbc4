"""Psd plugin -- Welch power spectral density of the accelerometer and gyroscope channels
(input ['fs','accel','gyro'], output ['algo_freq','psd_accel','psd_gyro']), with the semantics of
scipy.signal.welch; the estimator itself is csrc/welch_kernel.cuh (K11)."""
import numpy as np

from . import engine


class Psd(object):
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
        self.input = ['fs', 'accel', 'gyro']
        self.output = ['algo_freq', 'psd_accel', 'psd_gyro']
        self.batch = True
        self.results = None

    def run(self, set_of_input):
        '''
        set_of_input = [fs, accel (n,3), gyro (n,3)]
        '''
        fs = set_of_input[0]
        freq, p_a, p_g = self.run_batch(fs, np.asarray(set_of_input[1])[None], np.asarray(set_of_input[2])[None])
        self.results = [freq, p_a[0], p_g[0]]

    def run_batch(self, fs, accel, gyro, to_host=True, channel_major=False):
        '''
        accel, gyro: [R, n, 3] (the reference's per-run arrays, read in place) or, channel_major, [R, 3, n].
        Returns freq [L], psd_accel [R, L, 3], psd_gyro [R, L, 3], L = nperseg // 2 + 1.
        '''
        a = engine.to_device(accel)
        g = engine.to_device(gyro)
        w = engine.to_device(self.window, a.device)
        out = []
        for x in (a, g):
            if channel_major:
                R, _, n = x.shape
                kw = {}
            else:
                R, n, _ = x.shape
                kw = dict(inner=3, outer_stride=3 * n, sample_stride=3)
            if n < self.nperseg:
                raise ValueError('a series of %d samples is shorter than nperseg=%d' % (n, self.nperseg))
            psd, freq = engine.welch(fs, x, n, R * 3, self.nperseg, self.noverlap, w, **kw)
            out.append(psd.reshape(R, 3, -1).permute(0, 2, 1).contiguous())
        if to_host:
            return freq.cpu().numpy(), out[0].cpu().numpy(), out[1].cpu().numpy()
        return freq, out[0], out[1]

    def frequencies(self, fs):
        '''freq [L] of run_batch for sample rate fs: k / (nperseg (1/fs)), as np.fft.rfftfreq.'''
        return np.arange(self.nperseg // 2 + 1) * (1.0 / (self.nperseg * (1.0 / fs)))

    def get_results(self):
        return self.results

    def reset(self):
        pass
