"""Allan plugin -- device-backed mirror of demo_algorithms/allan_analysis.py:15-61
(input ['fs','accel','gyro'], output ['algo_time','ad_accel','ad_gyro']); the variance
itself is csrc/allan_kernel.cuh (K4, allan.allan_var allan.py:18-59) or, overlapping,
csrc/oallan_kernel.cuh (K4o); fit=True adds the IEEE Std 952 noise terms of every curve
(csrc/allanfit_kernel.cuh, K13) as ['noise_accel','noise_gyro'].  Hadamard: the overlapping Hadamard deviation on the same
tau grid (K4o's Hadamard form), output ['algo_time','hd_accel','hd_gyro']."""
import numpy as np
import torch

from . import engine
from .series_analysis import SeriesEstimator


class Allan(SeriesEstimator):
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

    fit=True also identifies the IEEE Std 952-1997 noise terms of every curve on the device (engine.allan_fit,
    K13), from the variance before its square root: outputs noise_accel and noise_gyro, [R, 3, 6] from run_batch
    and [3, 6] per run, rows the axes x, y, z and columns
        Q      quantisation                      rad            (accel m/s)
        N      angle / velocity random walk      rad/s/sqrt(Hz) (m/s^2/sqrt(Hz)), the IMU model's arw / vrw
        B      bias instability                  rad/s          (m/s^2)
        K      rate random walk                  rad/s^2/sqrt(Hz) (m/s^3/sqrt(Hz))
        R      rate ramp                         rad/s^2        (m/s^3)
        B_min  minimum deviation / 0.664         rad/s          (m/s^2), the datasheet bias-instability figure.
    The fit is the weighted non-negative least-squares fit of sigma^2 = sum_p C_p tau^p (p = -2..2) with relative
    residuals, each bin weighted by floor(n / m) - 1, the number of squared differences allan_var averages there.
    The overlapping curve is fitted with the same weights: it has more degrees of freedom than that at long tau,
    so for it the weights are a conservative proxy, not its degrees of freedom.
    '''

    def __init__(self, overlapping=False, fit=False):
        if not isinstance(overlapping, (bool, np.bool_)):
            raise TypeError('overlapping must be True or False, got %r' % (overlapping,))
        if not isinstance(fit, (bool, np.bool_)):
            raise TypeError('fit must be True or False, got %r' % (fit,))
        super().__init__(['algo_time', 'ad_accel', 'ad_gyro'] + (['noise_accel', 'noise_gyro'] if fit else []))
        self.overlapping = bool(overlapping)
        self.fit = bool(fit)

    @property
    def fused(self):
        return not self.overlapping     # engine.allan_mc: K1 fused into K4

    def _series(self, fs, x, n, nseries, **addressing):
        var, tau = self._variance()(fs, x, n, nseries, **addressing)
        if self.fit:
            return torch.sqrt(var), tau, engine.allan_fit(fs, n, var)
        return torch.sqrt(var), tau     # the DEVIATION, as allan_analysis.py:47-49

    def _variance(self):
        return engine.oallan if self.overlapping else engine.allan

    def abscissa(self, n, fs):
        return engine.allan_taus(n, fs)

    def run_bytes(self, n):
        # 64 B per run-sample for K1's series (48 B) and K4's workspace; K4o adds its prefix workspace for the
        # three series of one sensor
        return 64 + engine.oallan_workspace_bytes(n, 3) / n if self.overlapping else 64


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
