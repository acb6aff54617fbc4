"""Run-to-run bias, scale-factor and misalignment errors of the IMU error model in NumPy: the oracle of K1's and
K9's _rx forms (b2ins_imu_noise_rx_f64, b2ins_imu_err_stats_rx_f64) and of the run-error table
(b2ins_imu_run_err_f64), on top of noise952_np.imu_noise with the same draws.

Per sensor s (0 accel, 1 gyro) and run r, from the 1-sigma values of an imu_model dict ('b_std' [3], 'sf' [3],
'ma' a scalar for every off-diagonal or 3x3 with a zero diagonal; absent = 0), drawn once per run:
    (z0, z1) = normal_pair(t = 0xFFFFFFFD, id 44 + 6 s + j, run)
    j = 0..2:  b_run[j] = b_std[j] z0,  S[j][j] = sf[j] z1
    j = 3..5:  the off-diagonals of row i = j - 3 in column order: S[i][c0] = ma[i][c0] z0, S[i][c1] = ma[i][c1] z1
and every sample of the run gains delta[c] = b_run[c] + sum_j S[c][j] ref[j] (the kernel: d = b_run, then
d = fma(S[c][j], ref[j], d) for j = 0, 1, 2; the products here round once more, within 1e-16 of |S ref|).
"""
import numpy as np

import noise952_np as nz
import oracle_np as onp

DRAW_RUN_ERR = 44           # +6*sensor+j
RUN_ERR_T = 0xFFFFFFFD      # the counter word t of every run-error draw
RUN_ERR_KEYS = ('b_std', 'sf', 'ma')
# (row, column) of the two off-diagonals pair j = 3 + row fills, in column order
OFF_DIAG = ((1, 2), (0, 2), (0, 1))


def set_run_errors(err):
    return [k for k in RUN_ERR_KEYS if k in err and np.any(np.asarray(err[k], dtype=np.float64) != 0.0)]


def sigmas(err):
    """(b [3], sf [3], ma [3, 3]) of an imu_model dict, absent keys zero."""
    b = np.broadcast_to(np.asarray(err.get('b_std', 0.0), dtype=np.float64), (3,))
    sf = np.broadcast_to(np.asarray(err.get('sf', 0.0), dtype=np.float64), (3,))
    ma = np.asarray(err.get('ma', 0.0), dtype=np.float64)
    ma = ma * (1.0 - np.eye(3)) if ma.ndim == 0 else ma.reshape(3, 3)
    return b, sf, ma


def table(err, sensor, seed, run_ids):
    """[R, 3, 4] of one sensor: row i = (S[i][0], S[i][1], S[i][2], b_run[i])."""
    b, sf, ma = sigmas(err)
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    out = np.zeros((run_ids.size, 3, 4))
    for j in range(6):
        z0, z1 = onp.normal_pair(np.uint64(RUN_ERR_T), np.uint64(DRAW_RUN_ERR + 6 * sensor + j), run_ids, seed)
        if j < 3:
            out[:, j, 3] = b[j] * z0
            out[:, j, j] = sf[j] * z1
        else:
            i = j - 3
            c0, c1 = OFF_DIAG[i]
            out[:, i, c0] = ma[i, c0] * z0
            out[:, i, c1] = ma[i, c1] * z1
    return out


def delta(ref, tab):
    """delta [R, n, 3] = b_run + S ref of every run of tab [R, 3, 4] on ref [n, 3], in the kernel's order."""
    d = np.broadcast_to(tab[:, None, :, 3], (tab.shape[0], ref.shape[0], 3)).copy()
    for j in range(3):
        d = d + tab[:, None, :, j] * ref[None, :, j:j + 1]
    return d


def imu_noise(fs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_ids, vib_acc=None, vib_gyro=None):
    """noise952_np.imu_noise plus delta: gyro, accel [R, n, 3]."""
    gyro, accel = nz.imu_noise(fs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_ids, vib_acc, vib_gyro)
    if set_run_errors(gyro_err):
        gyro = gyro + delta(ref_gyro, table(gyro_err, 1, seed, run_ids))
    if set_run_errors(accel_err):
        accel = accel + delta(ref_accel, table(accel_err, 0, seed, run_ids))
    return gyro, accel
