"""MagCal plugin -- device-backed mirror of demo_algorithms/mag_calibrate.py:21-112 (input ['mag'], output
['soft_iron', 'hard_iron', 'mag_cal']); the calibration itself is csrc/magcal_kernel.cuh (K10, MagCalibrate,
MagCalibration.c:34-306)."""
import numpy as np

from . import engine


def check_segments(segments, n=None):
    """The segments as a (3, 2) int64 array.  ValueError unless they are three (start, end) pairs of integer
    row indices with end - start >= 3 and start >= 0 and, given the sample count n, end <= n."""
    if segments is None:
        raise ValueError('MagCal needs segments=((x0, xf), (y0, yf), (z0, zf)): the sample ranges of the '
                         'rotations about the x, y and z axes')
    try:
        seg = np.array(segments, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError('segments must be ((x0, xf), (y0, yf), (z0, zf)), got %r' % (segments,))
    if seg.shape != (3, 2) or not np.all(np.isfinite(seg)) or not np.all(seg == np.floor(seg)):
        raise ValueError('segments must be three (start, end) pairs of integer sample indices, got %r'
                         % (segments,))
    seg = seg.astype(np.int64)
    for a, b in seg:
        if a < 0 or b - a < 3 or (n is not None and b > n):
            raise ValueError('segment (%d, %d) must hold at least 3 samples inside [0, %s)'
                             % (a, b, 'n' if n is None else n))
    return seg


class MagCal(object):
    '''
    Soft- and hard-iron calibration of a magnetometer from three rotations of the sensor, about its x, y and
    z axes, in a uniform field.

    segments = ((x0, xf), (y0, yf), (z0, zf)): the half-open sample ranges of the three rotations (the six
    indices the reference asks for at its prompts; here they are required and nothing is plotted).  Each
    range holds at least 3 samples.  Outputs per run, with the reference's shapes:
        soft_iron (3, 3): S,
        hard_iron (1, 4): the hard iron and the estimated field magnitude [uT],
        mag_cal (L, 3):   the three segments stacked, each sample S m - hard_iron[0:3].
    A singular fit (for example noise-free samples from a plane through the origin) gives NaN in all of
    soft_iron and hard_iron.  Each segment is calibrated from its own samples: unlike the reference's
    wrapper, which corrects the rows of overlapping segments in place once per segment, overlapping ranges
    see the measured samples.
    '''

    def __init__(self, segments=None):
        self.segments = check_segments(segments)
        self.input = ['mag']
        self.output = ['soft_iron', 'hard_iron', 'mag_cal']
        self.batch = True
        self.results = None

    def run(self, set_of_input):
        '''
        set_of_input = [mag (n, 3)]
        '''
        mag = np.asarray(set_of_input[0], dtype=np.float64)
        si, hi, cal = self.run_batch(mag[None])
        self.results = [si[0], hi[0].reshape(1, 4), cal[0]]

    def run_batch(self, mag, to_host=True):
        '''
        mag: [R, n, 3] (numpy or a CUDA tensor).  Returns soft_iron [R, 3, 3], hard_iron [R, 4] and mag_cal
        [R, L, 3] (numpy, or CUDA tensors with to_host=False).
        '''
        shape = tuple(mag.shape)
        if len(shape) != 3 or shape[2] != 3:
            raise ValueError('mag must be [R, n, 3], got %s' % (shape,))
        check_segments(self.segments, shape[1])
        x = engine.to_device(mag)
        res = engine.mag_calibrate(self.segments, x, want_cal=True)
        if to_host:
            return res.soft_iron.cpu().numpy(), res.hard_iron.cpu().numpy(), res.mag_cal.cpu().numpy()
        return res.soft_iron, res.hard_iron, res.mag_cal

    def get_results(self):
        return self.results

    def reset(self):
        pass
