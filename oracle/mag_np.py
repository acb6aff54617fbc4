"""NumPy restatement of the magnetometer measurement generator (pathgen.mag_gen, pathgen.py:643-661) on
the b2ins noise spec, on top of oracle_np.  Test infrastructure only.

Draw ids (DESIGN.md section 4; csrc/common.cuh kDrawMag): the Box-Muller pair (k, 13, run) gives the
x and y normals of sample k, z0 of the pair (k, 14, run) the z normal.
"""
import numpy as np

from oracle_np import normal_pair

PAIR_MAG = 13       # (x, y); PAIR_MAG + 1: z from z0


def mag_normals(n, run_ids, seed):
    """[R, n, 3] normals of pathgen.mag_gen, in the order np.random.randn(n, 3) hands them out."""
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    k = np.arange(n, dtype=np.uint64)[None, :]
    z = np.empty((run_ids.size, n, 3))
    z[:, :, 0], z[:, :, 1] = normal_pair(k, PAIR_MAG, run_ids[:, None], seed)
    z[:, :, 2], _ = normal_pair(k, PAIR_MAG + 1, run_ids[:, None], seed)
    return z


def mag_gen(ref_mag, mag_err, z):
    """pathgen.mag_gen with the normals z [R, n, 3]: (ref_mag + hi) si^T + std z, in the reference's
    operation order.  ref_mag [n, 3] -> [R, n, 3]."""
    mea = (np.asarray(ref_mag, dtype=np.float64) + mag_err['hi']).dot(np.asarray(mag_err['si']).T)
    return mea[None] + np.asarray(mag_err['std']) * z
