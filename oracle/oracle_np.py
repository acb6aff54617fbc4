"""
ORACLE (test infrastructure, not product): NumPy restatement of the Monte-Carlo
free-integration hot path of gnss-ins-sim.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module, and only as the checker.  The product path
(gnss_ins_sim_b200) never imports anything under oracle/.

Every function cites the reference file:line (relative to the gnss-ins-sim
checkout) whose arithmetic it restates.  All arithmetic is float64; runs are
vectorised (axis 0 = run) while the time loop stays serial exactly like the
reference's (the recurrence is nonlinear in the state).

Pinned by tests/test_oracle_golden.py against tests/golden/*.npz, which were
produced by running the UNMODIFIED reference (oracle/gen_golden.py).

The device noise stream is defined here too (Philox4x32-10 + Box-Muller, the
"b2ins noise spec" of DESIGN.md section 4): the reference never seeds its RNG
(SURVEY 3.3), so "identical seeded draws" means: the device stream is the source
of truth and gen_golden.py injects THIS stream into the reference's
np.random.randn call sequence.
"""
import math

import numpy as np

# --------------------------------------------------------------------------
# WGS-84 constants, geoparams.py:18-23 and :40-43
# --------------------------------------------------------------------------
RE = 6378137.0
FLATTENING = 1.0 / 298.257223563
ECC = 0.0818191908426215
E_SQR = ECC ** 2
W_IE = 7292115e-11
NORMAL_GRAVITY = 9.7803253359
K_GRAV = 0.00193185265241
M_GRAV = 0.00344978650684

PI = math.pi
TWO_PI = 2.0 * math.pi
HALF_PI = 0.5 * math.pi


def geo_param(lat, h):
    """geoparams.geo_param, geoparams.py:25-53 (vectorised over runs)."""
    sl = np.sin(lat)
    cl = np.cos(lat)
    sl_sqr = sl * sl
    rm = (RE * (1 - E_SQR)) / (np.sqrt(1.0 - E_SQR * sl_sqr) * (1.0 - E_SQR * sl_sqr))
    rn = RE / (np.sqrt(1.0 - E_SQR * sl_sqr))
    g1 = NORMAL_GRAVITY * (1 + K_GRAV * sl_sqr) / np.sqrt(1.0 - E_SQR * sl_sqr)
    g = g1 * (1.0 - (2.0 / RE) * (1.0 + FLATTENING + M_GRAV - 2.0 * FLATTENING * sl_sqr) * h
              + 3.0 * h * h / RE / RE)
    return rm, rn, g, sl, cl


def lla2ecef(lla):
    """geoparams.lla2ecef, geoparams.py:70-87; lla[..., 3] -> xyz[..., 3]."""
    lla = np.asarray(lla, dtype=np.float64)
    sl = np.sin(lla[..., 0])
    cl = np.cos(lla[..., 0])
    sl_sqr = sl * sl
    r = RE / np.sqrt(1.0 - E_SQR * sl_sqr)
    rho = (r + lla[..., 2]) * cl
    x = rho * np.cos(lla[..., 1])
    y = rho * np.sin(lla[..., 1])
    z = (r * (1.0 - E_SQR) + lla[..., 2]) * sl
    return np.stack([x, y, z], axis=-1)


def euler2dcm_zyx(att):
    """attitude.euler2dcm 'zyx' branch, attitude.py:361-371.
    att[R,3] = [yaw, pitch, roll] -> c[R,3,3] (n -> b)."""
    c0, c1, c2 = np.cos(att[:, 0]), np.cos(att[:, 1]), np.cos(att[:, 2])
    s0, s1, s2 = np.sin(att[:, 0]), np.sin(att[:, 1]), np.sin(att[:, 2])
    c = np.empty((att.shape[0], 3, 3))
    c[:, 0, 0] = c1 * c0
    c[:, 0, 1] = c1 * s0
    c[:, 0, 2] = -s1
    c[:, 1, 0] = s2 * s1 * c0 - c2 * s0
    c[:, 1, 1] = s2 * s1 * s0 + c2 * c0
    c[:, 1, 2] = c1 * s2
    c[:, 2, 0] = s1 * c2 * c0 + s0 * s2
    c[:, 2, 1] = s1 * c2 * s0 - c0 * s2
    c[:, 2, 2] = c1 * c2
    return c


def euler_update_zyx(x, w, dt):
    """attitude.euler_update_zyx, attitude.py:679-721 (vectorised over runs).
    Forward Euler on the ZYX Euler-angle rates, pitch reflection at +-pi/2,
    then ONE +-2pi wrap of yaw and roll (not a modulo)."""
    c_psi = np.cos(x[:, 2])
    s_psi = np.sin(x[:, 2])
    t = w[:, 2] * c_psi + w[:, 1] * s_psi
    phi_dot = t / np.cos(x[:, 1])
    theta_dot = w[:, 1] * c_psi - w[:, 2] * s_psi
    psi_dot = w[:, 0] + t * np.tan(x[:, 1])
    y = x.copy()
    y[:, 0] += phi_dot * dt
    y[:, 1] += theta_dot * dt
    y[:, 2] += psi_dot * dt
    hi = y[:, 1] > HALF_PI
    lo = y[:, 1] < -HALF_PI
    y[hi, 1] = PI - y[hi, 1]
    y[lo, 1] = -PI - y[lo, 1]
    flip = hi | lo
    y[flip, 0] += PI
    y[flip, 2] += PI
    for k in (0, 2):
        up = y[:, k] > PI
        dn = y[:, k] < -PI
        y[up, k] -= TWO_PI
        y[dn, k] += TWO_PI
    return y


def cross3(a, b):
    """attitude.cross3, attitude.py:758-770."""
    return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1],
                     a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                     a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], axis=1)


def _mv(c, v):
    return np.einsum('rij,rj->ri', c, v)


def _mtv(c, v):
    return np.einsum('rji,rj->ri', c, v)


def free_integration(ref_frame, fs, gyro, accel, ini, earth_rot=True):
    """FreeIntegration.run, demo_algorithms/free_integration.py:63-174, batched.

    gyro, accel: [R, n, 3].  ini: [R, 9] or [R, 10] (row 9 = gravity override,
    free_integration.py:59-61) -- the caller has already applied the
    run_times -> idx selection of free_integration.py:85-87.
    Returns att, pos, vel: [R, n, 3].
    """
    gyro = np.asarray(gyro, dtype=np.float64)
    accel = np.asarray(accel, dtype=np.float64)
    ini = np.asarray(ini, dtype=np.float64)
    R, n, _ = accel.shape
    dt = 1.0 / fs
    att = np.zeros((R, n, 3))
    pos = np.zeros((R, n, 3))
    vel = np.zeros((R, n, 3))
    vel_b = np.zeros((R, n, 3))
    has_g = ini.shape[1] > 9
    r0, v0, att0 = ini[:, 0:3], ini[:, 3:6], ini[:, 6:9]
    att[:, 0] = att0
    vel_b[:, 0] = v0
    c_bn = euler2dcm_zyx(att[:, 0])
    vel[:, 0] = _mtv(c_bn, vel_b[:, 0])
    if ref_frame == 1:
        # free_integration.py:83-116
        g_n = np.zeros((R, 3))
        g_n[:, 2] = ini[:, 9] if has_g else geo_param(r0[:, 0], r0[:, 2])[2]
        pos[:, 0] = lla2ecef(r0)
        for i in range(1, n):
            att[:, i] = euler_update_zyx(att[:, i - 1], gyro[:, i - 1], dt)
            vel_b[:, i] = vel_b[:, i - 1] + (accel[:, i - 1] + _mv(c_bn, g_n)) * dt - \
                cross3(gyro[:, i - 1], vel_b[:, i - 1]) * dt
            c_bn = euler2dcm_zyx(att[:, i])
            vel[:, i] = _mtv(c_bn, vel_b[:, i])
            pos[:, i] = pos[:, i - 1] + vel[:, i - 1] * dt
    else:
        # free_integration.py:117-172
        pos[:, 0] = r0
        w_en_n = np.zeros((R, 3))
        w_ie_n = np.zeros((R, 3))
        g_n = np.zeros((R, 3))
        for i in range(1, n):
            rm, rn, g, sl, cl = geo_param(pos[:, i - 1, 0], pos[:, i - 1, 2])
            rm_e = rm + pos[:, i - 1, 2]
            rn_e = rn + pos[:, i - 1, 2]
            g_n[:, 2] = ini[:, 9] if has_g else g
            w_en_n[:, 0] = vel[:, i - 1, 1] / rn_e
            w_en_n[:, 1] = -vel[:, i - 1, 0] / rm_e
            w_en_n[:, 2] = -vel[:, i - 1, 1] * sl / cl / rn_e
            if earth_rot:
                w_ie_n[:, 0] = W_IE * cl
                w_ie_n[:, 2] = -W_IE * sl
            w_nb_b = gyro[:, i - 1] - _mv(c_bn, w_en_n + w_ie_n)
            att[:, i] = euler_update_zyx(att[:, i - 1], w_nb_b, dt)
            vel_dot_n = _mtv(c_bn, accel[:, i - 1]) + g_n - \
                cross3(2 * w_ie_n + w_en_n, vel[:, i - 1])
            vel[:, i] = vel[:, i - 1] + vel_dot_n * dt
            pos[:, i, 0] = pos[:, i - 1, 0] + vel[:, i - 1, 0] / rm_e * dt
            pos[:, i, 1] = pos[:, i - 1, 1] + vel[:, i - 1, 1] / rn_e / cl * dt
            pos[:, i, 2] = pos[:, i - 1, 2] + (-vel[:, i - 1, 2]) * dt
            c_bn = euler2dcm_zyx(att[:, i])
            vel_b[:, i] = _mv(c_bn, vel[:, i])
    return att, pos, vel


def free_integration_odo(ref_frame, fs, gyro, odo, ini, earth_rot=True):
    """free_integration_odo.FreeIntegration.run, demo_algorithms/free_integration_odo.py:63-160,
    batched: same attitude recurrence, body velocity = [odo, 0, 0].  gyro [R,n,3], odo [R,n]."""
    gyro = np.asarray(gyro, dtype=np.float64)
    odo = np.asarray(odo, dtype=np.float64)
    ini = np.asarray(ini, dtype=np.float64)
    R, n, _ = gyro.shape
    dt = 1.0 / fs
    att = np.zeros((R, n, 3))
    pos = np.zeros((R, n, 3))
    vel = np.zeros((R, n, 3))
    vel_b = np.zeros((R, 3))
    att[:, 0] = ini[:, 6:9]
    vel_b[:] = ini[:, 3:6]
    c_bn = euler2dcm_zyx(att[:, 0])
    vel[:, 0] = _mtv(c_bn, vel_b)
    pos[:, 0] = lla2ecef(ini[:, 0:3]) if ref_frame == 1 else ini[:, 0:3]
    w_en_n = np.zeros((R, 3))
    w_ie_n = np.zeros((R, 3))
    for i in range(1, n):
        if ref_frame == 1:
            att[:, i] = euler_update_zyx(att[:, i - 1], gyro[:, i - 1], dt)       # :104
        else:
            rm, rn, g, sl, cl = geo_param(pos[:, i - 1, 0], pos[:, i - 1, 2])    # :124-131
            rm_e = rm + pos[:, i - 1, 2]
            rn_e = rn + pos[:, i - 1, 2]
            w_en_n[:, 0] = vel[:, i - 1, 1] / rn_e
            w_en_n[:, 1] = -vel[:, i - 1, 0] / rm_e
            w_en_n[:, 2] = -vel[:, i - 1, 1] * sl / cl / rn_e
            if earth_rot:
                w_ie_n[:, 0] = W_IE * cl
                w_ie_n[:, 2] = -W_IE * sl
            w_nb_b = gyro[:, i - 1] - _mv(c_bn, w_en_n + w_ie_n)
            att[:, i] = euler_update_zyx(att[:, i - 1], w_nb_b, dt)
        vel_b[:, 0] = odo[:, i - 1]                                               # :106-108 / :142-144
        vel_b[:, 1] = 0.0
        vel_b[:, 2] = 0.0
        c_bn = euler2dcm_zyx(att[:, i])
        vel[:, i] = _mtv(c_bn, vel_b)
        if ref_frame == 1:
            pos[:, i] = pos[:, i - 1] + vel[:, i - 1] * dt                        # :112
        else:
            pos[:, i, 0] = pos[:, i - 1, 0] + vel[:, i - 1, 0] / rm_e * dt        # :149-154
            pos[:, i, 1] = pos[:, i - 1, 1] + vel[:, i - 1, 1] / rn_e / cl * dt
            pos[:, i, 2] = pos[:, i - 1, 2] + (-vel[:, i - 1, 2]) * dt
    return att, pos, vel


def gps_normals(m, run_ids, seed):
    """[R, m, 6] normals of pathgen.gps_gen: pairs (k, PAIR_GPS + j), j = 0..2, flattened."""
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    k = np.arange(m, dtype=np.uint64)[None, :]
    z = np.empty((run_ids.size, m, 6))
    for j in range(3):
        z0, z1 = normal_pair(k, PAIR_GPS + j, run_ids[:, None], seed)
        z[:, :, 2 * j] = z0
        z[:, :, 2 * j + 1] = z1
    return z


def gps_gen(ref_gps, gps_err, gps_type, z):
    """pathgen.gps_gen, pathgen.py:596-625.  ref_gps [m, 6]; z [R, m, 6] -> [R, m, 6]."""
    ref_gps = np.asarray(ref_gps, dtype=np.float64)
    pos_err = np.array(gps_err['stdp'], dtype=np.float64).copy()
    if gps_type == 0:
        rm, rn, _, _, cl = geo_param(ref_gps[0, 0], ref_gps[0, 2])
        pos_err[0] = pos_err[0] / rm
        pos_err[1] = pos_err[1] / rn / cl
    sd = np.concatenate([pos_err, np.asarray(gps_err['stdv'], dtype=np.float64)])
    return ref_gps[None, :, :] + sd[None, None, :] * z


def odo_normals(n, run_ids, seed):
    """[R, n] normals of pathgen.odo_gen: z0 of the pair (t, PAIR_ODO)."""
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    t = np.arange(n, dtype=np.uint64)[None, :]
    z0, _ = normal_pair(t, PAIR_ODO, run_ids[:, None], seed)
    return z0


def odo_gen(ref_odo, odo_err, z):
    """pathgen.odo_gen, pathgen.py:627-641: scale*ref + stdv*randn(n).  z [R, n]."""
    return odo_err['scale'] * np.asarray(ref_odo)[None, :] + odo_err['stdv'] * z


# --------------------------------------------------------------------------
# b2ins noise spec: Philox4x32-10 (Salmon et al. SC'11; same constants and
# round schedule as cuRAND / torch) + Box-Muller in float64.
# --------------------------------------------------------------------------
_M0 = np.uint64(0xD2511F53)
_M1 = np.uint64(0xCD9E8D57)
_W0 = 0x9E3779B9
_W1 = 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)

# Philox counter word 1: which draw of (run, t) this is.
PAIR_ACCEL = 0      # +axis : (GM drive, white) of accel axis
PAIR_GYRO = 3       # +axis : (GM drive, white) of gyro axis
PAIR_VIB = 6        # +axis : (accel random vib, gyro random vib)
PAIR_PHASE = 9      # +axis, t = 0xFFFFFFFF : sinusoidal gyro-vib phase uniforms
PAIR_ODO = 12       # odometer white noise (z0)
PAIR_PSD = 16       # +3*sensor+axis (sensor 0 accel, 1 gyro), t = bin index: PSD phases (z0)
PAIR_GPS = 24       # +j, t = GPS sample: (pos0, pos1), (pos2, vel0), (vel1, vel2)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """All arguments broadcastable integer arrays/scalars (taken mod 2^32).
    Returns four uint64 arrays holding 32-bit words."""
    c0 = np.asarray(c0, dtype=np.uint64) & _MASK
    c1 = np.asarray(c1, dtype=np.uint64) & _MASK
    c2 = np.asarray(c2, dtype=np.uint64) & _MASK
    c3 = np.asarray(c3, dtype=np.uint64) & _MASK
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0 = int(k0) & 0xFFFFFFFF
    k1 = int(k1) & 0xFFFFFFFF
    for _ in range(10):
        p0 = _M0 * c0
        p1 = _M1 * c2
        hi0, lo0 = p0 >> _S32, p0 & _MASK
        hi1, lo1 = p1 >> _S32, p1 & _MASK
        c0, c1, c2, c3 = (hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0)
        k0 = (k0 + _W0) & 0xFFFFFFFF
        k1 = (k1 + _W1) & 0xFFFFFFFF
    return c0, c1, c2, c3


def normal_pair(t, pair, run, seed):
    """Two independent N(0,1) float64 for (run, t, pair) under `seed`.

    counter = (t, pair, run_lo, run_hi), key = (seed_lo, seed_hi).
    u1 = 1 - (x1:x0 >> 12) * 2^-52 in (0, 1],  u2 = (x3:x2 >> 12) * 2^-52 in [0, 1)
    (both exact in float64; the device builds them from the bit pattern).
    r = sqrt(-2 ln u1);  z0 = r cos(2 pi u2), z1 = r sin(2 pi u2).
    """
    run = np.asarray(run, dtype=np.uint64)
    seed = int(seed)
    x0, x1, x2, x3 = philox4x32_10(t, pair, run & _MASK, run >> _S32,
                                   seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    a = (x1 << _S32) | x0
    b = (x3 << _S32) | x2
    u1 = 1.0 - (a >> np.uint64(12)).astype(np.float64) * (2.0 ** -52)
    u2 = (b >> np.uint64(12)).astype(np.float64) * (2.0 ** -52)
    r = np.sqrt(-2.0 * np.log(u1))
    th = TWO_PI * u2
    return r * np.cos(th), r * np.sin(th)


def noise_normals(n, run_ids, seed):
    """The per-(run, t) normals the device draws.
    Returns dict of [R, n, 3] arrays: acc_gm, acc_w, gyr_gm, gyr_w."""
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    t = np.arange(n, dtype=np.uint64)[None, :, None]
    ax = np.arange(3, dtype=np.uint64)[None, None, :]
    r = run_ids[:, None, None]
    acc_gm, acc_w = normal_pair(t, PAIR_ACCEL + ax, r, seed)
    gyr_gm, gyr_w = normal_pair(t, PAIR_GYRO + ax, r, seed)
    return {'acc_gm': acc_gm, 'acc_w': acc_w, 'gyr_gm': gyr_gm, 'gyr_w': gyr_w}


def vib_normals(n, run_ids, seed):
    """Random-vibration normals: (accel vib, gyro vib), each [R, n, 3]."""
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    t = np.arange(n, dtype=np.uint64)[None, :, None]
    ax = np.arange(3, dtype=np.uint64)[None, None, :]
    return normal_pair(t, PAIR_VIB + ax, run_ids[:, None, None], seed)


def gyro_vib_phase_uniforms(run_ids, seed):
    """Uniform [0,1) phases of pathgen.py:553-555 (np.random.rand(1) per axis): [R,3]."""
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    ax = np.arange(3, dtype=np.uint64)[None, :]
    r = run_ids[:, None]
    seed = int(seed)
    x0, x1, _, _ = philox4x32_10(0xFFFFFFFF, PAIR_PHASE + ax, r & _MASK, r >> _S32,
                                 seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    a = (x1 << _S32) | x0
    return (a >> np.uint64(12)).astype(np.float64) * (2.0 ** -52)


def psd_phase_normals(L, run_ids, seed, sensor):
    """The L random-phase normals of each (run, axis) PSD series: z0 of the pair
    (t = k, draw = PAIR_PSD + 3*sensor + axis).  Returns [R, 3, L]."""
    run_ids = np.asarray(run_ids, dtype=np.uint64)
    k = np.arange(L, dtype=np.uint64)[None, None, :]
    ax = np.arange(3, dtype=np.uint64)[None, :, None]
    z0, _ = normal_pair(k, PAIR_PSD + 3 * sensor + ax, run_ids[:, None, None], seed)
    return z0


def gm_coeffs(corr, drift, fs):
    """pathgen.bias_drift coefficients, pathgen.py:583-586: a is the first-order
    approximation 1 - dt/tau, b uses the exact exponential -- both as written."""
    corr = np.asarray(corr, dtype=np.float64)
    drift = np.asarray(drift, dtype=np.float64)
    with np.errstate(divide='ignore', invalid='ignore'):
        a = 1 - 1 / fs / corr
        b = drift * np.sqrt(1.0 - np.exp(-2 / (fs * corr)))
    return a, b


def bias_drift(corr, drift, n, fs, z):
    """pathgen.bias_drift, pathgen.py:565-594, with the normals supplied.
    z[R, n, 3]: z[:, j, i] drives d[:, j+1, i] (GM) or IS d[:, j, i]/drift (corr=inf)."""
    R = z.shape[0]
    d = np.zeros((R, n, 3))
    a, b = gm_coeffs(corr, drift, fs)
    for i in range(3):
        if not math.isinf(corr[i]):
            for j in range(1, n):
                d[:, j, i] = a[i] * d[:, j - 1, i] + b[i] * z[:, j - 1, i]
        else:
            d[:, :, i] = drift[i] * z[:, :, i]
    return d


def sensor_gen(fs, ref, err, white_key, z_gm, z_w, vib=None):
    """pathgen.acc_gen / gyro_gen, pathgen.py:441-501 / :503-563:
    meas = ref + b + drift + white + vib  (summed in that order, pathgen.py:500,562)."""
    n = ref.shape[0]
    dt = 1.0 / fs
    drift = bias_drift(err['b_corr'], err['b_drift'], n, fs, z_gm)
    white = z_w.copy()
    for c in range(3):
        white[:, :, c] = err[white_key][c] / math.sqrt(dt) * white[:, :, c]
    out = ref[None] + np.asarray(err['b'], dtype=np.float64) + drift + white
    if vib is not None:
        out = out + vib
    else:
        out = out + np.zeros((n, 3))
    return out


def sinusoidal_vib(fs, n, amp, freq, phase=None):
    """pathgen.py:490-493 (accel, zero phase) / :553-555 (gyro, random phase)."""
    dt = 1.0 / fs
    k = np.arange(n)
    out = np.empty((1 if phase is None else phase.shape[0], n, 3))
    for c in range(3):
        ph = 0.0 if phase is None else (phase[:, c] * 2 * PI)[:, None]
        out[:, :, c] = amp[c] * np.sin(2.0 * PI * freq * dt * k[None, :] + ph)
    return out


def imu_noise(fs, ref_gyro, ref_accel, gyro_err, accel_err, seed, run_ids,
              vib_acc=None, vib_gyro=None):
    """Loop A of Sim.__gen_data_from_pathgen, ins_sim.py:490-496, for the runs in
    run_ids, with the b2ins noise stream.  Returns gyro, accel [R, n, 3].
    vib_*: None or dict(type='random'|'sinusoidal', x,y,z[,freq]) (ins_sim.py:642-701)."""
    n = ref_accel.shape[0]
    z = noise_normals(n, run_ids, seed)
    va = vg = None
    if vib_acc is not None or vib_gyro is not None:
        zva, zvg = vib_normals(n, run_ids, seed)
    if vib_acc is not None:
        amp = np.array([vib_acc['x'], vib_acc['y'], vib_acc['z']], dtype=np.float64)
        if vib_acc['type'] == 'random':
            va = zva * amp
        elif vib_acc['type'] == 'sinusoidal':
            va = sinusoidal_vib(fs, n, amp, vib_acc['freq'])
    if vib_gyro is not None:
        amp = np.array([vib_gyro['x'], vib_gyro['y'], vib_gyro['z']], dtype=np.float64)
        if vib_gyro['type'] == 'random':
            vg = zvg * amp
        elif vib_gyro['type'] == 'sinusoidal':
            vg = sinusoidal_vib(fs, n, amp, vib_gyro['freq'],
                                gyro_vib_phase_uniforms(run_ids, seed))
    accel = sensor_gen(fs, ref_accel, accel_err, 'vrw', z['acc_gm'], z['acc_w'], va)
    gyro = sensor_gen(fs, ref_gyro, gyro_err, 'arw', z['gyr_gm'], z['gyr_w'], vg)
    return gyro, accel


# --------------------------------------------------------------------------
# error statistics, ins_data_manager.py
# --------------------------------------------------------------------------
def angle_range_pi(x):
    """attitude.angle_range_pi, attitude.py:799-812 (python float % semantics)."""
    x = np.mod(x, TWO_PI)
    return np.where(x > PI, x - TWO_PI, x)


def array_error(x, r, angle=False):
    """InsDataMgr.array_error lla==0 branch, ins_data_manager.py:536-541."""
    err = x - r
    return angle_range_pi(err) if angle else err


def array_stats(x):
    """InsDataMgr.__array_stats, ins_data_manager.py:797-808 (np.std ddof=0)."""
    return {'max': np.max(np.abs(x), 0), 'avg': np.average(x, 0), 'std': np.std(x, 0)}


def end_point_error_stats(att, pos, vel, ref_att, ref_pos, ref_vel):
    """get_error_stats(err_stats_start=-1) for att_euler (angle), pos, vel:
    ins_data_manager.py:385-452, :717-759.  Inputs [R,n,3] and refs [n,3]."""
    return {'att_euler': array_stats(array_error(att[:, -1], ref_att[-1], True)),
            'pos': array_stats(array_error(pos[:, -1], ref_pos[-1])),
            'vel': array_stats(array_error(vel[:, -1], ref_vel[-1]))}


def process_error_stats(x, ref, start_idx, angle=False):
    """__process_error_stats, ins_data_manager.py:761-795: per-run stats over
    samples idx >= start_idx.  x[R,n,3], ref[n,3] -> dict of [R,3]."""
    err = array_error(x[:, start_idx:], ref[None, start_idx:], angle)
    return {'max': np.max(np.abs(err), 1), 'avg': np.average(err, 1), 'std': np.std(err, 1)}


# --------------------------------------------------------------------------
# Allan variance, allan.py:18-59
# --------------------------------------------------------------------------
def allan_multipliers(n, fs):
    """allan.py:29-44: bin sizes m = j*10^k (j=1..9), m <= floor(n/9)."""
    ts = 1.0 / fs
    max_bin = int(math.floor(n / 9.0))
    if max_bin * ts < 1:
        return []
    mult = []
    nextpow10 = math.ceil(math.log10(max_bin))
    scale = 0.1
    for _ in range(nextpow10):
        scale *= 10
        for j in range(1, 10):
            tmp = int(j * scale)
            if tmp <= max_bin:
                mult.append(tmp)
            else:
                break
    return mult


def allan_var(x, fs):
    """allan.allan_var, allan.py:18-59.  Returns (avar, tau)."""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    mult = allan_multipliers(n, fs)
    if not mult:
        return np.array([]), np.array([])
    ts = 1.0 / fs
    avar = np.zeros(len(mult))
    tau = np.zeros(len(mult))
    for i, m in enumerate(mult):
        nb = n // m
        if nb < 9:
            break
        means = np.mean(x[:nb * m].reshape(nb, m), 1)
        d = means[1:] - means[:-1]
        avar[i] = 0.5 / (nb - 1) * np.sum(d * d)
        tau[i] = m * ts          # allan.py:58 (not m / fs: the two differ in the last bit)
    return avar, tau


# --------------------------------------------------------------------------
# PSD vibration, psd/time_series_from_psd.py:17-65
# --------------------------------------------------------------------------
def psd_bins(sxx, freq, fs, n, phase_normals):
    """The period N and the L = N/2 + 1 complex bins xk = A + jB that time_series_from_psd
    transforms (time_series_from_psd.py:36-54); None if the table exceeds fs/2."""
    sxx = np.array(sxx, dtype=np.float64)
    freq = np.asarray(freq, dtype=np.float64)
    if fs < 2.0 * freq[-1] or fs < 0.0:
        return None
    N = n
    if n % 2 != 0:
        N = n + 1
    if N > 16384:
        N = 16384
    L = freq.shape[0]
    if L != N // 2 + 1:
        L = N // 2 + 1
        sxx = np.interp(np.linspace(0, fs / 2.0, L), freq, sxx)
    sxx[1:L - 1] = 0.5 * sxx[1:L - 1]
    ax = np.sqrt(sxx * N * fs)
    phi = PI * np.asarray(phase_normals, dtype=np.float64)[:L]
    return N, ax * np.exp(1j * phi)


def tile_period(xt, n):
    """A series of period N = len(xt) for n samples, as time_series_from_psd.py:58-63 repeats it."""
    N = xt.shape[0]
    return np.hstack([np.tile(xt, (n // N,)), xt[0:n % N]]) if n != N else xt


def time_series_from_psd(sxx, freq, fs, n, phase_normals):
    """time_series_from_psd with the L random-phase normals supplied (first-call
    behaviour: the caller's sxx is NOT halved in place, see SURVEY 7 'quirks')."""
    bins = psd_bins(sxx, freq, fs, n, phase_normals)
    if bins is None:
        return False, np.zeros((n,))
    N, xk = bins
    xk = np.hstack([xk, xk[-2:0:-1].conj()])
    xt = np.fft.ifft(xk).real
    return True, tile_period(xt, n)
