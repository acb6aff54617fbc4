"""ORACLE (test infrastructure) -- the loosely-coupled filter (ekf_np.ins_loose) initialising itself from its
measurements: InsLoose(align_yaw=...) (DESIGN.md section 11, "Alignment").

The reference's InsLoose.ins_loose (demo_algorithms/ins_loose.py:54-126) is the only part of that stub with
logic: it averages the first samples_for_attitude_ini = 10 accelerometer samples (:73-79), takes pitch and
roll from the normalised mean (:80-91: pitch = asin(a_x), roll = atan2(-a_y, -a_z); yaw is a placeholder,
10 deg), and takes position and velocity from the latest GPS row at or before that sample, else from the first
one after it, propagating the attitude until then (:92-119).  Here:
  1. levelling at sample N-1 from the mean of accel[0..N-1] (the measurements the filter reads); yaw is the
     given align_yaw, or with 'gps' the course over ground atan2(v_E, v_N) of the fix row's GPS velocity;
  2. the fix row: the latest VISIBLE GPS row at or before sample N-1, else the first visible row after it;
     the filter starts at s0 = max(N-1, gps_idx[fix]) with position and velocity as measured there;
  3. between N-1 and s0 the attitude alone propagates (euler_update_zyx on the gyro: no Earth or transport
     rate, no bias estimate, no covariance);
  4. P0 at s0 per run, diagonal (p0_aligned); no initial-state draw;
  5. from s0 the filter of ekf_np.ins_loose runs unchanged; its first update is the first visible row after
     s0.  History rows before the state exists are NaN (attitude before N-1, position and velocity before
     s0; wb, ab are 0 there); the consistency record takes epochs after s0.

ekf_np.ins_loose starts from one shared initial state and covariance, so the filter loop from s0 is restated
here (ekf_np's prediction, six scalar updates, correction and consistency record, line for line) for a per-run
initial state and P0.  ins_loose filters given measurements (the fed form); ins_loose_gen generates them as
ekf_np / ekf_vib_np do (oracle_np.sensor_gen with each sensor's vibration, oracle_np.gps_gen) and adds the
bias truth the consistency record needs.
"""
import numpy as np

import ekf_np
import ekf_vib_np
import oracle_np as onp

N_ALIGN = 10           # ins_loose.py:72 samples_for_attitude_ini
G_LEVEL = 9.80665      # the specific force the levelling P0 divides by [m/s^2]
MIN_SPEED = 1.0        # 'gps' heading: the least horizontal speed at the fix row [m/s]


def fix_row(gps_idx, gps_vis, n=N_ALIGN):
    """The GPS row that starts the filter: the latest visible row with gps_idx <= n-1, else the first visible
    row after n-1; None without a visible row."""
    gps_idx, gps_vis = np.asarray(gps_idx).reshape(-1), np.asarray(gps_vis).reshape(-1)
    vis = np.nonzero(gps_vis > 0)[0]
    if vis.size == 0:
        return None
    before = vis[gps_idx[vis] <= n - 1]
    return int(before[-1]) if before.size else int(vis[0])


def start_sample(gps_idx, j, n=N_ALIGN):
    """First sample with a full state: max(N-1, the fix row's sample)."""
    return max(n - 1, int(np.asarray(gps_idx).reshape(-1)[j]))


def level(accel, n=N_ALIGN):
    """[R] pitch, roll from the mean of accel[:, 0..N-1] (ins_loose.py:76-91, summed in sample order)."""
    s = np.zeros((accel.shape[0], 3))
    for i in range(n):
        s = s + accel[:, i]
    a = s / float(n)
    norm = np.sqrt(a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1] + a[:, 2] * a[:, 2])
    a = a / norm[:, None]
    return np.arcsin(a[:, 0]), np.arctan2(-a[:, 1], -a[:, 2])


def course(gps_vel):
    """[R] course over ground atan2(v_E, v_N) of GPS velocities [R, 2] (v_N, v_E)."""
    return np.arctan2(gps_vel[:, 1], gps_vel[:, 0])


def p0_aligned(fs, gyro_err, accel_err, gps_err, ini_att_std, gap, gps_vel=None, n=N_ALIGN):
    """[R or 1, 15] diagonal P0 at the start sample.  Position, velocity: stdp^2, stdv^2.  Level misalignment N
    (set by roll, accelerometer y) and E (set by pitch, accelerometer x): (b^2 + b_drift^2 + vrw^2 fs / N) / g^2.
    Yaw: ini_att_std[2]^2 for a given heading; with gps_vel [R, 2] (the fix row's v_N, v_E) the course variance
    (stdv_N^2 v_E^2 + stdv_E^2 v_N^2) / |v_h|^4.  The attitude block grows over the propagation gap [s] by
    arw^2 gap + (b^2 + b_drift^2) gap^2 (gyro axis c for attitude c).  Biases: ekf_np.default_p0's."""
    base = ekf_np.default_p0(gyro_err, accel_err, gps_err, ini_att_std)
    ab, ad, vrw = (np.asarray(accel_err[k], dtype=np.float64) for k in ('b', 'b_drift', 'vrw'))
    lev = (ab * ab + ad * ad + vrw * vrw * float(fs) / n) / (G_LEVEL * G_LEVEL)
    gb, gd, arw = (np.asarray(gyro_err[k], dtype=np.float64) for k in ('b', 'b_drift', 'arw'))
    grow = arw * arw * gap + (gb * gb + gd * gd) * (gap * gap)
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


def check(n, gps_idx, gps_vis, align_yaw, gps_vel_rows):
    """The host checks of an aligned launch (ValueError): a series shorter than N, no visible GPS row, and with
    'gps' a horizontal speed below MIN_SPEED at the fix row.  gps_vel_rows: [R, m, 2] or [m, 2] GPS v_N, v_E.
    Returns (fix row, start sample)."""
    if n < N_ALIGN:
        raise ValueError('alignment needs at least %d IMU samples (got %d)' % (N_ALIGN, n))
    j = fix_row(gps_idx, gps_vis)
    if j is None:
        raise ValueError('alignment needs a visible GPS row')
    if align_yaw == 'gps':
        v = np.asarray(gps_vel_rows, dtype=np.float64)[..., j, :]
        if not np.all(np.hypot(v[..., 0], v[..., 1]) >= MIN_SPEED):
            raise ValueError("align_yaw='gps' needs a horizontal speed of at least %g m/s at the fix row" % MIN_SPEED)
    return j, start_sample(gps_idx, j)


def ins_loose(fs, gyro, accel, gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err, align_yaw,
              ini_att_std=(0.02, 0.005, 0.005), earth_rot=True, ref_nav=None, bias_g=None, bias_a=None,
              stats_start=0, want_hist=False, vel_rw=0.0, att_rw=0.0):
    """The aligned filter on measurements gyro, accel [R, n, 3], gps [R, m, 6].  align_yaw: a heading [rad] or
    'gps'.  ref_nav [n, 9] (optional): end_err; with bias_g, bias_a [R, n, 3] (the true biases) also the
    consistency record of the epochs after the start sample with i >= stats_start.  Returns ekf_np.ins_loose's
    dict plus 'fix_row', 'start', 'p0' [R, 15]."""
    gyro, accel, gps = (np.asarray(a, dtype=np.float64) for a in (gyro, accel, gps))
    gps_idx, gps_vis = np.asarray(gps_idx).reshape(-1), np.asarray(gps_vis).reshape(-1)
    R, n = gyro.shape[:2]
    dt = 1.0 / fs
    jf, s0 = check(n, gps_idx, gps_vis, align_yaw, gps[:, :, 3:5])
    fx = gps[:, jf]
    # ---- 1. levelling at N-1 -------------------------------------------------------------------------
    pitch, roll = level(accel)
    if align_yaw == 'gps':
        yaw = course(fx[:, 3:5])
        p0 = p0_aligned(fs, gyro_err, accel_err, gps_err, ini_att_std, (s0 - (N_ALIGN - 1)) * dt, fx[:, 3:5])
    else:
        yaw = np.full(R, float(align_yaw))
        p0 = np.tile(p0_aligned(fs, gyro_err, accel_err, gps_err, ini_att_std, (s0 - (N_ALIGN - 1)) * dt), (R, 1))
    att = np.stack([yaw, pitch, roll], 1)
    hist = None
    if want_hist:
        hist = {k: np.full((R, n, 3), np.nan) for k in ('att', 'pos', 'vel')}
        hist.update({k: np.zeros((R, n, 3)) for k in ('wb', 'ab')})
    # ---- 3. attitude alone from N-1 to s0 ------------------------------------------------------------------
    for i in range(N_ALIGN - 1, s0):
        if want_hist:
            hist['att'][:, i] = att
        att = onp.euler_update_zyx(att, gyro[:, i], dt)
    # ---- 2, 4. the state at s0 ---------------------------------------------------------------------------
    pos, vel = fx[:, 0:3].copy(), fx[:, 3:6].copy()
    P = np.einsum('ri,ij->rij', p0, np.eye(15))
    # ---- 5. ekf_np.ins_loose's filter from s0, first update at the first row after s0 -----------------------------
    att, pos, vel, bg, ba, P, acc = filter_from(fs, gyro, accel, gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err,
                                                s0, int(np.searchsorted(gps_idx, s0, side='right')), att, pos, vel,
                                                P, hist, earth_rot, ref_nav, bias_g, bias_a, stats_start, vel_rw,
                                                att_rw)
    consist = ref_nav is not None and bias_g is not None
    out = {'end_bias': np.concatenate([bg, ba], 1), 'P_diag_end': np.einsum('rii->ri', P), 'fix_row': jf,
           'start': s0, 'p0': p0}
    if ref_nav is not None:
        end = ref_nav[n - 1]
        out['end_err'] = np.concatenate([onp.angle_range_pi(att - end[0:3]), pos - end[3:6], vel - end[6:9]], 1)
    if consist:
        cnt = max(acc['cnt'], 1)
        out.update({'nees': acc['nees'] / cnt, 'inside3': acc['inside'] / cnt, 'epochs': acc['cnt']})
    if want_hist:
        out.update(hist)
    return out


def ins_loose_gen(fs, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err,
                  seed, run_ids, align_yaw, vib_acc=None, vib_gyro=None, want_imu=False, **kw):
    """The aligned filter on the measurements a generated experiment makes for run_ids under seed (those of
    ekf_np.ins_loose; with vib_acc / vib_gyro those of ekf_vib_np.ins_loose), with the consistency record.
    kw: ins_loose's ini_att_std, earth_rot, stats_start, want_hist, vel_rw, att_rw."""
    run_ids = np.asarray(run_ids)
    n, m = ref_gyro.shape[0], np.asarray(ref_gps).shape[0]
    z = onp.noise_normals(n, run_ids, seed)
    accel = onp.sensor_gen(fs, ref_accel, accel_err, 'vrw', z['acc_gm'], z['acc_w'],
                           ekf_vib_np.vibration(fs, n, run_ids, seed, vib_acc, 0))
    gyro = onp.sensor_gen(fs, ref_gyro, gyro_err, 'arw', z['gyr_gm'], z['gyr_w'],
                          ekf_vib_np.vibration(fs, n, run_ids, seed, vib_gyro, 1))
    bias_g = np.asarray(gyro_err['b'])[None, None] + onp.bias_drift(gyro_err['b_corr'], gyro_err['b_drift'], n, fs, z['gyr_gm'])
    bias_a = np.asarray(accel_err['b'])[None, None] + onp.bias_drift(accel_err['b_corr'], accel_err['b_drift'], n, fs, z['acc_gm'])
    gps = onp.gps_gen(ref_gps, gps_err, 0, onp.gps_normals(m, run_ids, seed))
    out = ins_loose(fs, gyro, accel, gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err, align_yaw,
                    ref_nav=np.asarray(ref_nav, dtype=np.float64), bias_g=bias_g, bias_a=bias_a, **kw)
    if want_imu:
        out.update({'gyro': gyro, 'accel': accel, 'gps': gps})
    return out


def filter_from(fs, gyro, accel, gps, gps_idx, gps_vis, gyro_err, accel_err, gps_err, s0, j0, att, pos, vel, P, hist=None,
                earth_rot=True, ref_nav=None, bias_g=None, bias_a=None, stats_start=0, vel_rw=0.0, att_rw=0.0):
    """ekf_np.ins_loose's filter loop (prediction, six scalar updates, correction, consistency record), restated
    line for line for a per-run initial state att, pos, vel [R, 3] and P [R, 15, 15] at sample s0, with GPS rows
    from j0; zero bias estimates.  hist (dict of [R, n, 3], or None) is filled from row s0.  From s0 = j0 = 0 at
    ekf_np's initial state this is ekf_np.ins_loose bit for bit (tests/test_cpu_ekf_align.py).  Returns att, pos,
    vel, bg, ba, P at the last sample and the consistency accumulators {'nees', 'inside', 'cnt'}."""
    R, n, m, dt = gyro.shape[0], gyro.shape[1], gps.shape[1], 1.0 / fs
    want_hist = hist is not None
    a_g, b_g = onp.gm_coeffs(gyro_err['b_corr'], gyro_err['b_drift'], fs)
    a_a, b_a = onp.gm_coeffs(accel_err['b_corr'], accel_err['b_drift'], fs)
    white_g = np.isinf(np.asarray(gyro_err['b_corr'], dtype=np.float64))
    white_a = np.isinf(np.asarray(accel_err['b_corr'], dtype=np.float64))
    a_g, b_g = np.where(white_g, 0.0, a_g), np.where(white_g, np.asarray(gyro_err['b_drift']), b_g)
    a_a, b_a = np.where(white_a, 0.0, a_a), np.where(white_a, np.asarray(accel_err['b_drift']), b_a)
    arw2 = np.asarray(gyro_err['arw'], dtype=np.float64) ** 2
    vrw2 = np.asarray(accel_err['vrw'], dtype=np.float64) ** 2
    r_diag = np.concatenate([np.asarray(gps_err['stdp'], dtype=np.float64) ** 2,
                             np.asarray(gps_err['stdv'], dtype=np.float64) ** 2])
    bg, ba = np.zeros((R, 3)), np.zeros((R, 3))
    consist = ref_nav is not None and bias_g is not None
    acc = {'nees': np.zeros((R, 3)), 'inside': np.zeros((R, 15)), 'cnt': 0}
    skew = ekf_np.skew
    I15 = np.eye(15)
    j = j0
    for i in range(s0, n):
        if j < m and gps_idx[j] == i:
            if gps_vis[j] > 0:
                rm, rn, _, _, cl = onp.geo_param(pos[:, 0], pos[:, 2])
                zm = np.empty((R, 6))
                zm[:, 0] = (pos[:, 0] - gps[:, j, 0]) * (rm + pos[:, 2])
                zm[:, 1] = (pos[:, 1] - gps[:, j, 1]) * (rn + pos[:, 2]) * cl
                zm[:, 2] = -(pos[:, 2] - gps[:, j, 2])
                zm[:, 3:6] = vel - gps[:, j, 3:6]
                x = np.zeros((R, 15))
                for k in range(6):
                    s = P[:, k, k] + r_diag[k]
                    K = P[:, :, k] / s[:, None]
                    x = x + K * (zm[:, k] - x[:, k])[:, None]
                    P = P - K[:, :, None] * P[:, k, None, :]
                    P = 0.5 * (P + np.transpose(P, (0, 2, 1)))
                pos[:, 0] -= x[:, 0] / (rm + pos[:, 2])
                pos[:, 1] -= x[:, 1] / ((rn + pos[:, 2]) * cl)
                pos[:, 2] += x[:, 2]
                vel = vel - x[:, 3:6]
                c_nb = np.einsum('rij,rjk->rik', onp.euler2dcm_zyx(att), np.eye(3)[None] - skew(x[:, 6:9]))
                att = ekf_np.dcm2euler_zyx(c_nb)
                bg = bg - x[:, 9:12]
                ba = ba - x[:, 12:15]
            if consist and i >= stats_start:
                rm, rn, _, _, cl = onp.geo_param(ref_nav[i, 3], ref_nav[i, 5])
                e = np.zeros((R, 15))
                e[:, 0] = (pos[:, 0] - ref_nav[i, 3]) * (rm + ref_nav[i, 5])
                e[:, 1] = (pos[:, 1] - ref_nav[i, 4]) * (rn + ref_nav[i, 5]) * cl
                e[:, 2] = -(pos[:, 2] - ref_nav[i, 5])
                e[:, 3:6] = vel - ref_nav[i, 6:9]
                mm = np.einsum('rji,rjk->rik', onp.euler2dcm_zyx(att), onp.euler2dcm_zyx(np.tile(ref_nav[i, 0:3], (R, 1))))
                e[:, 6] = -0.5 * (mm[:, 2, 1] - mm[:, 1, 2])
                e[:, 7] = -0.5 * (mm[:, 0, 2] - mm[:, 2, 0])
                e[:, 8] = -0.5 * (mm[:, 1, 0] - mm[:, 0, 1])
                e[:, 9:12] = bg - bias_g[:, i]
                e[:, 12:15] = ba - bias_a[:, i]
                for b in range(3):
                    blk = slice(3 * b, 3 * b + 3)
                    acc['nees'][:, b] += np.einsum('ri,rij,rj->r', e[:, blk], np.linalg.inv(P[:, blk, blk]), e[:, blk])
                acc['inside'] += (np.abs(e) <= 3.0 * np.sqrt(np.einsum('rii->ri', P)))
                acc['cnt'] += 1
            j += 1
        if want_hist:
            hist['att'][:, i], hist['pos'][:, i], hist['vel'][:, i] = att, pos, vel
            hist['wb'][:, i], hist['ab'][:, i] = bg, ba
        if i == n - 1:
            break
        w = gyro[:, i] - bg
        f = accel[:, i] - ba
        c_nb = onp.euler2dcm_zyx(att)
        f_n = onp._mtv(c_nb, f)
        c_bn = np.transpose(c_nb, (0, 2, 1))
        Phi = np.tile(I15, (R, 1, 1))
        Phi[:, 0:3, 3:6] = np.eye(3) * dt
        Phi[:, 3:6, 6:9] = skew(f_n) * dt
        Phi[:, 3:6, 12:15] = -c_bn * dt
        Phi[:, 6:9, 9:12] = c_bn * dt
        Phi[:, 9:12, 9:12] = np.diag(a_g)
        Phi[:, 12:15, 12:15] = np.diag(a_a)
        Q = np.zeros((R, 15, 15))
        Q[:, 3:6, 3:6] = np.einsum('rij,j,rkj->rik', c_bn, vrw2, c_bn) * dt + np.eye(3) * (vel_rw * vel_rw * dt)
        Q[:, 6:9, 6:9] = np.einsum('rij,j,rkj->rik', c_bn, arw2, c_bn) * dt + np.eye(3) * (att_rw * att_rw * dt)
        Q[:, 9:12, 9:12] = np.diag(b_g ** 2)
        Q[:, 12:15, 12:15] = np.diag(b_a ** 2)
        P = np.einsum('rij,rjk,rlk->ril', Phi, P, Phi) + Q
        att, pos, vel = ekf_np.nav_step_rf0(att, pos, vel, w, f, dt, earth_rot)
        bg = bg * a_g
        ba = ba * a_a
    return att, pos, vel, bg, ba, P, acc
