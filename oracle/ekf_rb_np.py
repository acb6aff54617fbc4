"""ORACLE (test infrastructure) -- the loosely-coupled filter spec with a run-to-run turn-on bias (DESIGN.md
section 11, "Turn-on bias"; ekf_kernel<..., RB>).

Every run draws b_run[c] = b_std[c] z0 of run-error pair c of its sensor (run_err_np.table: the draw K1-rx and
b2ins_imu_run_err_f64 make for the same global run), and its measurements carry the constant bias b + b_run.  The
filter's model knows the spread: P0 of the bias states is b_drift^2 + b^2 + b_std^2, and the aligned level and gap
terms add b_std^2 to b^2 + b_drift^2 (default_p0, p0_aligned); Q is unchanged.  The consistency record's true bias
is b + (b_run + d), d the Gauss-Markov drift (the kernel forms (b + b_run) + d: the same bits when b = 0).

The filter loops are those of ekf_np.ins_loose (ekf_vib_np's measurements with vibration), ekf_align_np.ins_loose
and ekf_fed_np.ins_loose, run unchanged: this module hands them the measurements with the folded bias and the truth
with b_run, and swaps ekf_np.default_p0 / ekf_align_np.p0_aligned for the ones above during the call, as ekf_vib_np
and ekf_fed_np swap ekf_np's generators.  The generated forms return that oracle's dict plus end_bias_err [R, 6]:
the gyro then accel bias estimates minus the true biases at n-1.  With b_std absent or zero every output of those
oracles is unchanged, bit for bit.
"""
import contextlib

import numpy as np

import ekf_align_np
import ekf_fed_np
import ekf_np
import ekf_vib_np
import oracle_np as onp
import run_err_np

_BASE_P0 = ekf_np.default_p0
N_ALIGN, G_LEVEL = ekf_align_np.N_ALIGN, ekf_align_np.G_LEVEL


def _b_std(err):
    return np.asarray(err['b_std'], dtype=np.float64) if 'b_std' in err else None


def turn_on_bias(err, sensor, seed, run_ids):
    """[R, 3] constant bias of every run's measurements of one sensor (0 accel, 1 gyro): the IMU's 'b' plus the
    run's b_run (the b_run column of Sim.imu_run_errors()); 'b' itself [3] without a non-zero 'b_std'."""
    b = np.asarray(err['b'], dtype=np.float64)
    if not np.any(np.asarray(err.get('b_std', 0.0), dtype=np.float64) != 0.0):
        return b
    return b + run_err_np.table(err, sensor, seed, run_ids)[:, :, 3]


def default_p0(gyro_err, accel_err, gps_err, ini_att_std):
    """ekf_np.default_p0 with b_std^2 added to the bias states: b_drift^2 + b^2 + b_std^2."""
    p0 = _BASE_P0(gyro_err, accel_err, gps_err, ini_att_std)
    for err, at in ((gyro_err, 9), (accel_err, 12)):
        s = _b_std(err)
        if s is not None:
            p0[at:at + 3] = p0[at:at + 3] + s ** 2
    return p0


def p0_aligned(fs, gyro_err, accel_err, gps_err, ini_att_std, gap, gps_vel=None, n=N_ALIGN):
    """ekf_align_np.p0_aligned with b_std^2 added to b^2 + b_drift^2 in the level term
    (b^2 + b_drift^2 + b_std^2 + vrw^2 fs / N) / g^2 and in the gyro's growth over the gap; biases: default_p0."""
    base = default_p0(gyro_err, accel_err, gps_err, ini_att_std)
    ab, ad, vrw = (np.asarray(accel_err[k], dtype=np.float64) for k in ('b', 'b_drift', 'vrw'))
    lev = ab * ab + ad * ad
    if _b_std(accel_err) is not None:
        lev = lev + _b_std(accel_err) ** 2
    lev = (lev + vrw * vrw * float(fs) / n) / (G_LEVEL * G_LEVEL)
    gb, gd, arw = (np.asarray(gyro_err[k], dtype=np.float64) for k in ('b', 'b_drift', 'arw'))
    gv = gb * gb + gd * gd
    if _b_std(gyro_err) is not None:
        gv = gv + _b_std(gyro_err) ** 2
    grow = arw * arw * gap + gv * (gap * gap)
    if gps_vel is None:
        yaw = np.full(1, base[8])
    else:
        sv = np.broadcast_to(np.asarray(gps_err['stdv'], dtype=np.float64), (3,))
        vn, ve = gps_vel[:, 0], gps_vel[:, 1]
        h2 = vn * vn + ve * ve
        yaw = (sv[0] * sv[0] * (ve * ve) + sv[1] * sv[1] * (vn * vn)) / (h2 * h2)
    p0 = np.tile(base, (yaw.size, 1))
    p0[:, 6] = lev[1] + grow[0]
    p0[:, 7] = lev[0] + grow[1]
    p0[:, 8] = yaw + grow[2]
    return p0


@contextlib.contextmanager
def _model(on=True):
    """ekf_np / ekf_align_np with this module's P0 (on) for the duration of the block."""
    saved = ekf_np.default_p0, ekf_align_np.p0_aligned
    if on:
        ekf_np.default_p0, ekf_align_np.p0_aligned = default_p0, p0_aligned
    try:
        yield
    finally:
        ekf_np.default_p0, ekf_align_np.p0_aligned = saved


def _b_run(err, sensor, seed, run_ids):
    """[R, 1, 3] b_run of one sensor, or None without a non-zero b_std."""
    if not np.any(np.asarray(err.get('b_std', 0.0), dtype=np.float64) != 0.0):
        return None
    return run_err_np.table(err, sensor, seed, run_ids)[:, None, :, 3]


class _BiasedOnp(object):
    """oracle_np as ekf_np.ins_loose sees it: sensor_gen folds each run's b_run into the constant bias (and adds the
    sensor's vibration last, as ekf_vib_np does), and the bias truth ekf_np forms as b + bias_drift(...) gets
    b_run + d.  Keys: 'vrw' accelerometer, 'arw' gyro (sensor_gen's white-noise key)."""

    def __init__(self, b_run, vib):
        self._b_run, self._vib = b_run, vib
        self.z, self.truth_part = None, {}

    def __getattr__(self, name):
        return getattr(onp, name)

    def noise_normals(self, n, run_ids, seed):
        self.z = onp.noise_normals(n, run_ids, seed)
        return self.z

    def sensor_gen(self, fs, ref, err, white_key, z_gm, z_w):
        br = self._b_run[white_key]
        if br is not None:
            err = dict(err, b=np.asarray(err['b'], dtype=np.float64) + br)
        return onp.sensor_gen(fs, ref, err, white_key, z_gm, z_w, self._vib[white_key])

    def bias_drift(self, corr, drift, n, fs, z):
        key = 'arw' if z is self.z['gyr_gm'] else 'vrw'
        d = onp.bias_drift(corr, drift, n, fs, z)
        if self._b_run[key] is not None:
            d = self._b_run[key] + d
        self.truth_part[key] = d
        return d


def ins_loose(fs, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err, seed,
              run_ids, ini, vib_acc=None, vib_gyro=None, model_b_std=True, **kw):
    """ekf_np.ins_loose (same arguments; kw: ini_att_std, earth_rot, stats_start, want_hist, vel_rw, att_rw) on
    measurements that carry each run's turn-on bias (and vib_acc / vib_gyro as ekf_vib_np.ins_loose takes them),
    with b_std in P0 (model_b_std False leaves it out: the filter of the parent model on the same data).  Adds
    end_bias_err [R, 6]."""
    n = np.asarray(ref_gyro).shape[0]
    hook = _BiasedOnp({'vrw': _b_run(accel_err, 0, seed, run_ids), 'arw': _b_run(gyro_err, 1, seed, run_ids)},
                      {'vrw': ekf_vib_np.vibration(fs, n, run_ids, seed, vib_acc, 0),
                       'arw': ekf_vib_np.vibration(fs, n, run_ids, seed, vib_gyro, 1)})
    saved = ekf_np.onp
    ekf_np.onp = hook
    try:
        with _model(model_b_std):
            out = ekf_np.ins_loose(fs, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis, gyro_err, accel_err,
                                   gps_err, seed, run_ids, ini, **kw)
    finally:
        ekf_np.onp = saved
    truth = np.concatenate([np.asarray(gyro_err['b']) + hook.truth_part['arw'][:, n - 1],
                            np.asarray(accel_err['b']) + hook.truth_part['vrw'][:, n - 1]], axis=1)
    out['end_bias_err'] = out['end_bias'] - truth
    return out


def ins_loose_aligned(fs, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err,
                      seed, run_ids, align_yaw, vib_acc=None, vib_gyro=None, **kw):
    """ekf_align_np.ins_loose_gen (same arguments; kw: ekf_align_np.ins_loose's) on measurements that carry each
    run's turn-on bias, with p0_aligned.  Adds end_bias_err [R, 6]."""
    run_ids = np.asarray(run_ids)
    n, m = ref_gyro.shape[0], np.asarray(ref_gps).shape[0]
    z = onp.noise_normals(n, run_ids, seed)
    hook = _BiasedOnp({'vrw': _b_run(accel_err, 0, seed, run_ids), 'arw': _b_run(gyro_err, 1, seed, run_ids)},
                      {'vrw': ekf_vib_np.vibration(fs, n, run_ids, seed, vib_acc, 0),
                       'arw': ekf_vib_np.vibration(fs, n, run_ids, seed, vib_gyro, 1)})
    hook.z = z
    accel = hook.sensor_gen(fs, ref_accel, accel_err, 'vrw', z['acc_gm'], z['acc_w'])
    gyro = hook.sensor_gen(fs, ref_gyro, gyro_err, 'arw', z['gyr_gm'], z['gyr_w'])
    bias_g = np.asarray(gyro_err['b'])[None, None] + hook.bias_drift(gyro_err['b_corr'], gyro_err['b_drift'], n, fs,
                                                                     z['gyr_gm'])
    bias_a = np.asarray(accel_err['b'])[None, None] + hook.bias_drift(accel_err['b_corr'], accel_err['b_drift'], n,
                                                                      fs, z['acc_gm'])
    gps = onp.gps_gen(ref_gps, gps_err, 0, onp.gps_normals(m, run_ids, seed))
    with _model():
        out = ekf_align_np.ins_loose(fs, gyro, accel, gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err, align_yaw,
                                     ref_nav=np.asarray(ref_nav, dtype=np.float64), bias_g=bias_g, bias_a=bias_a, **kw)
    out['end_bias_err'] = out['end_bias'] - np.concatenate([bias_g[:, n - 1], bias_a[:, n - 1]], axis=1)
    return out


def ins_loose_fed(*args, **kw):
    """ekf_fed_np.ins_loose (same arguments) with b_std in P0: supplied measurements carry their bias already."""
    with _model():
        return ekf_fed_np.ins_loose(*args, **kw)
