"""What the series estimators (Allan, Hadamard, Psd) share: the reference's plugin protocol, and the device
front end that reads the three accelerometer and three gyroscope series of every run in place."""
import numpy as np

from . import engine


class SeriesEstimator(object):
    '''
    One statistic per accelerometer and gyroscope channel, on an abscissa that depends only on the series
    length and the sample rate (input ['fs', 'accel', 'gyro'], output [abscissa, accel statistic, gyro
    statistic], then the accel and gyro forms of any per-series outputs).  An estimator supplies _series (its
    device call on a batch of series), abscissa and run_bytes; fused is True where Sim may generate the series
    inside the estimator.
    '''
    fused = False

    def __init__(self, output):
        self.input = ['fs', 'accel', 'gyro']
        self.output = output
        self.batch = True
        self.results = None

    def run(self, set_of_input):
        '''
        set_of_input = [fs, accel (n,3), gyro (n,3)]
        '''
        fs = set_of_input[0]
        x, *per_run = self.run_batch(fs, np.asarray(set_of_input[1])[None], np.asarray(set_of_input[2])[None])
        self.results = [x] + [v[0] for v in per_run]

    def run_batch(self, fs, accel, gyro, to_host=True, channel_major=False):
        '''
        accel, gyro: [R, n, 3] (the reference's per-run arrays, 3R interleaved series read in place) or,
        channel_major, [R, 3, n] (3R contiguous series, which the estimators stream with bulk copies).
        Returns the abscissa [L], the accel and the gyro statistics [R, L, 3], then, for an estimator with
        per-series outputs [E] (Allan(fit=True)), their accel and gyro forms [R, 3, E] (rows: axes x, y, z).
        '''
        out, per_series = [], []
        for x in (engine.to_device(accel), engine.to_device(gyro)):
            if channel_major:
                R, _, n = x.shape
                kw = {}
            else:
                R, n, _ = x.shape
                kw = dict(inner=3, outer_stride=3 * n, sample_stride=3)
            y, abscissa, *extra = self._series(fs, x, n, R * 3, **kw)
            out.append(y.reshape(R, 3, -1).permute(0, 2, 1).contiguous())
            per_series += [e.reshape(R, 3, -1) for e in extra]
        res = [abscissa] + out + per_series
        return tuple(r.cpu().numpy() for r in res) if to_host else tuple(res)

    def _series(self, fs, x, n, nseries, **addressing):
        '''The statistic [nseries, L] and the abscissa [L] (CUDA) of nseries series of n samples in x, addressed
        as engine.allan addresses them; an estimator with per-series outputs returns them third, [nseries, E].'''
        raise NotImplementedError

    def abscissa(self, n, fs):
        '''The abscissa [L] of run_batch for series of n samples at fs, on the host.'''
        raise NotImplementedError

    def run_bytes(self, n):
        '''Device memory per run-sample when Sim generates the series of n samples and runs this estimator.'''
        raise NotImplementedError

    def get_results(self):
        return self.results

    def reset(self):
        pass
