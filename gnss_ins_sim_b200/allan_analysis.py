"""Allan plugin -- device-backed mirror of demo_algorithms/allan_analysis.py:15-61
(input ['fs','accel','gyro'], output ['algo_time','ad_accel','ad_gyro']); the variance
itself is csrc/allan_kernel.cuh (K4, allan.allan_var allan.py:18-59) or, overlapping,
csrc/oallan_kernel.cuh (K4o).  Hadamard: the overlapping Hadamard deviation on the same
tau grid (K4o's Hadamard form), output ['algo_time','hd_accel','hd_gyro']."""
import numpy as np
import torch

from . import engine


class Allan(object):
    '''
    Allan deviation of the three accelerometer and three gyroscope channels.

    overlapping=False (the default) is the reference's estimator, allan.allan_var: clusters of m
    samples start at multiples of m, so the longest cluster sizes average only a few differences.
    overlapping=True is the overlapping Allan variance of NIST SP 1065 (eq. 10) and IEEE Std 952:
    every start offset counts,
        avar(m) = 1 / (2 m^2 M) * sum_{k<M} (S(k+m, m) - S(k, m))^2,  M = n - 2m + 1,
    with S(k, m) the sum of the m samples from k.  It has many more degrees of freedom at long tau,
    where bias instability and rate random walk are read.  Both use the same tau grid
    (m = j*10^k <= n/9), so the two curves can be laid over each other.
    '''

    def __init__(self, overlapping=False):
        if not isinstance(overlapping, (bool, np.bool_)):
            raise TypeError('overlapping must be True or False, got %r' % (overlapping,))
        self.overlapping = bool(overlapping)
        self.input = ['fs', 'accel', 'gyro']
        self.output = ['algo_time', 'ad_accel', 'ad_gyro']
        self.batch = True
        self.results = None

    def run(self, set_of_input):
        '''
        set_of_input = [fs, accel (n,3), gyro (n,3)]
        '''
        fs = set_of_input[0]
        tau, ad_a, ad_g = self.run_batch(fs, np.asarray(set_of_input[1])[None],
                                         np.asarray(set_of_input[2])[None])
        self.results = [tau, ad_a[0], ad_g[0]]

    def run_batch(self, fs, accel, gyro, to_host=True, channel_major=False):
        '''
        accel, gyro: [R, n, 3] (the reference's per-run arrays) or, channel_major, [R, 3, n].
        Returns tau [ntau], ad_accel [R, ntau, 3], ad_gyro [R, ntau, 3]
        (Allan DEVIATION = sqrt(avar), allan_analysis.py:47-49).
        '''
        a = engine.to_device(accel)
        g = engine.to_device(gyro)
        var = self._variance()
        out = []
        for x in (a, g):
            if channel_major:     # 3R contiguous series: the bulk-copy front end of K4
                R, _, n = x.shape
                avar, tau = var(fs, x, n, R * 3)
            else:                 # 3R interleaved series, read in place (no copy)
                R, n, _ = x.shape
                avar, tau = var(fs, x, n, R * 3, inner=3, outer_stride=3 * n, sample_stride=3)
            out.append(torch.sqrt(avar).reshape(R, 3, -1).permute(0, 2, 1).contiguous())
        if to_host:
            return tau.cpu().numpy(), out[0].cpu().numpy(), out[1].cpu().numpy()
        return tau, out[0], out[1]

    def _variance(self):
        return engine.oallan if self.overlapping else engine.allan

    def get_results(self):
        return self.results

    def reset(self):
        pass


class Hadamard(Allan):
    '''
    Overlapping Hadamard deviation of the three accelerometer and three gyroscope channels
    (NIST SP 1065), on Allan's tau grid (m = j*10^k <= n/9):
        hvar(m) = 1 / (6 m^2 H) * sum_{k<H} (S(k+2m, m) - 2 S(k+m, m) + S(k, m))^2,  H = n - 3m + 1,
    with S(k, m) the sum of the m samples from k.  A second difference of adjacent cluster sums: a linear
    drift of the rate (thermal drift, the rate ramp R of IEEE Std 952), which adds b^2 tau^2 / 2 to the
    Allan variance and hides bias instability and rate random walk at long tau, cancels exactly.  White
    noise gives sigma^2 / m as the Allan variance does, so the two curves can be laid over each other.
    run / run_batch / get_results / reset as Allan's; the deviations are published as hd_accel and
    hd_gyro, never as ad_*.
    '''

    def __init__(self):
        super().__init__(overlapping=True)
        self.output = ['algo_time', 'hd_accel', 'hd_gyro']

    def _variance(self):
        return engine.ohadamard
