/*
 * b2ins -- H100-native Monte-Carlo strapdown-INS engine: C ABI.
 *
 * This is the drop-in boundary for the Monte-Carlo free-integration hot path of
 * gnss-ins-sim (SURVEY.md section 8b).  Every entry point names the reference
 * interface it replaces (file:line relative to the gnss-ins-sim checkout).
 *
 * Conventions
 *   - plain C, no torch / C++ types; all floating point is IEEE double ("f64").
 *   - functions return B2INS_OK (0) or an error code; b2ins_last_error() gives text
 *     (thread-local).  Nothing is allocated across the boundary: the caller owns
 *     every buffer.
 *   - entry points WITHOUT a suffix take DEVICE pointers and a CUDA stream
 *     (void* = cudaStream_t, NULL = legacy default stream) and are asynchronous.
 *   - entry points ending in _host take HOST pointers, do the H2D / D2H copies
 *     themselves on an internal stream and return when the results are in the
 *     caller's buffers (this is what a ctypes / cgo / JNI stub binds first).
 *   - series of per-run 3-vectors x(run r, sample t, component c) use one of these
 *     layouts:
 *       B2INS_LAYOUT_RUN_MAJOR  [R][n][3]  -- run r is exactly the reference's
 *                                             (n,3) C-contiguous numpy array
 *       B2INS_LAYOUT_TIME_MAJOR [n][3][R]  -- device-native for lanes_per_run = 1
 *       B2INS_LAYOUT_CHANNEL_MAJOR [R][3][n] -- every channel of every run a contiguous
 *                                             series (K1 output only: what K4 reads best)
 *   - "ini" is [ini_sets][ini_rows] (ini_rows = 9: lat,lon,alt [rad,rad,m], body
 *     velocity [m/s], yaw,pitch,roll [rad]; ini_rows = 10 adds a gravity override
 *     [m/s^2]) -- the transpose of FreeIntegration's ini_pos_vel_att
 *     (free_integration.py:19-61).  Global run g uses set g if g < ini_sets,
 *     else set 0 (free_integration.py:85-87).
 */
#ifndef B2INS_H_
#define B2INS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2INS_VERSION 100 /* 0.1.0 */

#define B2INS_OK 0
#define B2INS_ERR_ARG 1    /* bad argument (NULL, size, alignment, enum) */
#define B2INS_ERR_CUDA 2   /* a CUDA call or kernel failed */
#define B2INS_ERR_NODEV 3  /* no usable CUDA device */

#define B2INS_LAYOUT_RUN_MAJOR 0
#define B2INS_LAYOUT_TIME_MAJOR 1
#define B2INS_LAYOUT_CHANNEL_MAJOR 2

#define B2INS_VIB_NONE 0
#define B2INS_VIB_RANDOM 1     /* pathgen.py:486-489 / :549-552 */
#define B2INS_VIB_SINUSOIDAL 2 /* pathgen.py:490-493 / :553-555 (gyro: random phase) */
#define B2INS_VIB_SERIES 3     /* precomputed per-axis series (PSD model), see b2ins_psd_series_f64 */

/* Sensor error model of one triad: pathgen.acc_gen / gyro_gen `acc_err` / `gyro_err`
 * dicts (pathgen.py:441-466, :503-528), already in SI units as produced by
 * imu_model.IMU (imu_model.py:138-143). */
typedef struct b2ins_sensor_err {
  double b[3];       /* constant bias */
  double b_drift[3]; /* bias-instability 1-sigma */
  double b_corr[3];  /* Gauss-Markov correlation time [s]; +inf => white drift (pathgen.py:591-593) */
  double rw[3];      /* 'arw' [rad/s/sqrt(Hz)] or 'vrw' [m/s^2/sqrt(Hz)] */
} b2ins_sensor_err;

/* The IEEE Std 952 terms of one triad that b2ins_sensor_err does not hold (DESIGN.md section 4), in the units of
 * the Allan noise identification's columns Q, K and R (b2ins_allan_fit_f64).  Per axis c, sample t, dt = 1/fs:
 *   q: quantisation [rad; accel m/s]: e[t] = q sqrt(12) (u[t] - 1/2), u uniform in [0, 1); rate error (e[t+1] - e[t]) / dt
 *   k: rate random walk [rad/s^2/sqrt(Hz); accel m/s^3/sqrt(Hz)]: w[0] = 0, w[t+1] = w[t] + k sqrt(dt) z[t]
 *   r: rate ramp [rad/s^2; accel m/s^3]: r t dt, the same in every run
 * q and k must be finite and >= 0, r finite. */
typedef struct b2ins_noise_terms {
  double q[3];
  double k[3];
  double r[3];
} b2ins_noise_terms;

/* The run-to-run errors of one triad (DESIGN.md section 4): 1-sigma values in SI units, each drawn once per run
 * from the run's global id and constant over the run.  Per axis c of run r:
 *   b:  turn-on bias [rad/s; accel m/s^2]: b_run[c] = b[c] z, added to b2ins_sensor_err.b;
 *   sf: scale factor [-]: S[c][c] = sf[c] z;
 *   ma: misalignment [rad]: S[i][j] = ma[i][j] z (i != j), the sensitivity of sensor axis i to true axis j;
 *       the diagonal must be 0.
 * The measurement gains delta[c] = b_run[c] + sum_j S[c][j] ref[j]: M = I + S scales the true rate or specific
 * force, not the vibration.  Draws: counter t = 0xFFFFFFFD, id 44 + 6 sensor + j (sensor 0 accel, 1 gyro);
 * j = 0..2: (z0, z1) = (b_run[j], sf[j]); j = 3..5: the off-diagonals of row j - 3 in column order.
 * Every value must be finite and >= 0. */
typedef struct b2ins_run_err {
  double b[3];
  double sf[3];
  double ma[3][3];
} b2ins_run_err;

/* Vibration model of one triad: Sim.__parse_env output (ins_sim.py:642-701). */
typedef struct b2ins_vib {
  int32_t type; /* B2INS_VIB_* */
  int32_t series_len; /* VIB_SERIES: period of the series (<= 16384, it is tiled to n like
                         time_series_from_psd.py:59-62) */
  double amp[3];  /* RANDOM: 1-sigma; SINUSOIDAL: amplitude */
  double freq;    /* SINUSOIDAL: Hz */
  const double* series; /* VIB_SERIES: device pointer [runs][3][series_len], else NULL */
} b2ins_vib;

/* One Monte-Carlo experiment: loops A and B of Sim.run (ins_sim.py:490-506,
 * ins_algo_manager.py:73-95) for `runs` runs starting at global run id `run_offset`. */
typedef struct b2ins_mc_config {
  int32_t ref_frame;  /* 0 NED/LLA, 1 virtual inertial (free_integration.py:83,117) */
  int32_t earth_rot;  /* FreeIntegration(earth_rot=...), only used when ref_frame == 0 */
  double fs;          /* IMU sample rate [Hz] */
  int64_t n;          /* samples per run */
  int64_t runs;       /* runs computed by this call (this rank's shard) */
  int64_t run_offset; /* global id of local run 0: names the Philox stream of every run */
  int64_t ini_offset; /* local run r is simulation run ini_offset + r for the initial-state rule
                         (FreeIntegration.run_times, free_integration.py:85-87) */
  uint64_t seed;      /* Philox key */
  b2ins_sensor_err gyro_err;
  b2ins_sensor_err accel_err;
  b2ins_vib vib_gyro;
  b2ins_vib vib_accel;
  int32_t ini_sets;
  int32_t ini_rows;       /* 9 or 10 */
  int32_t lanes_per_run;  /* 0 = choose from runs; else 1,2,4,8,16,32 (32 = one warp owns one run) */
  int32_t stats_start;    /* first sample index of the per-run process-error statistics
                             (ins_data_manager.py:761-795); < 0 = end-point errors only */
  int64_t dump_runs;      /* full histories are written for local runs [0, dump_runs) */
  /* algorithm: 0 = FreeIntegration (free_integration.py), 1 = the odometer variant
   * (demo_algorithms/free_integration_odo.py:63-160: body velocity = [odometer, 0, 0]) with
   * pathgen.odo_gen noise (pathgen.py:627-641): odo = odo_scale*ref_odo + odo_stdv*randn */
  int32_t algo;
  int32_t dump_stride;    /* histories keep samples 0, s, 2s, ... (rows = ceil(n / s)); 0 and 1 = every
                             sample.  Decimated output for plotting error histories of many runs
                             (Sim.plot / results(err_stats_start >= 0) territory, ins_sim.py:253-315) */
  double odo_scale;
  double odo_stdv;
  const double* ref_odo;  /* algo 1: DEVICE pointer [n], true forward speed (pathgen 'odo') */
  double* dump_odo;       /* algo 1, nullable: DEVICE pointer [dump_runs][n] odometer histories */
  double* dump_quat;      /* nullable: DEVICE pointer [dump_runs][rows][4], the scalar-first quaternion of
                             every kept attitude sample -- the att_quat the reference associates with each
                             att_euler it holds (ins_sim.py:729-794, attitude.euler2quat :188-205) */
} b2ins_mc_config;

/* frame of the position columns of proc_stats, b2ins_mc_free_integration_ex_f64 */
#define B2INS_POS_FRAME_LLA 0   /* (lat, lon, alt) differences, as b2ins_mc_free_integration_f64 */
#define B2INS_POS_FRAME_NED 1   /* metres: the reference's get_error_stats(extra_opt='ned') */
#define B2INS_POS_FRAME_ECEF 2  /* metres: extra_opt='ecef' */

/* ---- K1 + K4 fused: the Allan experiment without the series ------------------------------------
 * Replaces, for a whole Monte-Carlo Allan experiment, pathgen.acc_gen / gyro_gen (pathgen.py:441-594)
 * followed by allan.allan_var (allan.py:18-59) per run and channel (Allan.run, allan_analysis.py:29-49):
 * every (run, channel) series is generated tile by tile inside the tau-binning kernel and never
 * written.  Series s = run * 6 + channel (accel x y z, gyro x y z).  No vibration models here (the
 * caller materialises the series with b2ins_imu_noise_f64 when env is set); n must exceed 5040.
 *   avar [runs * 6][ntau], tau [ntau]; workspace: b2ins_allan_workspace_bytes(n, runs * 6). */
int b2ins_allan_mc_f64(double fs, int64_t n, int64_t runs, const double* ref_gyro,
                       const double* ref_accel, const b2ins_sensor_err* gyro_err,
                       const b2ins_sensor_err* accel_err, uint64_t seed, int64_t run_offset,
                       double* avar, double* tau, void* workspace, void* stream);

/* ---- K7: loosely-coupled GNSS/INS filter (BASELINE config 5) ------------------------------------
 * Replaces demo_algorithms/ins_loose.py:54-138 (InsLoose.ins_loose / prediction / correction) -- which
 * in the reference is a stub: its prediction() and correction() are `pass`.  The filter here is a
 * 15-state closed-loop error-state EKF specified in DESIGN.md section 11 (parity with the reference is
 * unpinnable; the kernel is held to that spec and validated by NEES / 3-sigma tests), fed by the
 * reference's sensor models: pathgen.acc_gen / gyro_gen (pathgen.py:441-594) and gps_gen (:596-625)
 * on the same Philox streams as K12 / K6.  ref_frame 0 only (LLA positions, NED velocities). */
typedef struct {
  double fs;
  int64_t n;            /* IMU samples */
  int64_t runs;
  int64_t run_offset;   /* global id of local run 0 */
  int64_t m;            /* GPS samples */
  uint64_t seed;
  b2ins_sensor_err gyro_err;
  b2ins_sensor_err accel_err;
  double gps_stdp[3];   /* GPS position noise [m]: generator and filter R (imu_model gps_opt 'stdp') */
  double gps_stdv[3];   /* GPS velocity noise [m/s] */
  double ini[9];        /* true initial lat, lon [rad], alt [m], body velocity [m/s], yaw, pitch, roll [rad] */
  double ini_att_std[3];/* 1-sigma of the initial misalignment (N, E, D) [rad]; initial position / velocity
                           errors are drawn with the GPS sigmas, bias variances start at drift^2 + b^2 */
  int64_t stats_start;  /* first IMU sample index of the consistency record */
  int64_t dump_runs;    /* histories for local runs [0, dump_runs) */
  int32_t dump_stride;  /* keep samples 0, s, 2s, ... (0, 1 = all) */
  int32_t earth_rot;
  double vel_rw;        /* extra velocity random walk of the filter model [m/s/sqrt(s)]: covers the
                           mismatch between the reference's truth generator and its own first-order
                           mechanization (noise-free free integration of motion_def-ins.csv drifts by
                           0.37 m/s); 0.02 keeps the filter consistent on that trajectory */
  double att_rw;        /* extra misalignment random walk [rad/sqrt(s)] */
} b2ins_ekf_config;

/* One launch: every run generates its IMU and GPS measurements, filters them and leaves
 *   end_err   [runs][9]  att (wrapped), pos (LLA), vel error at sample n-1 (as K12's end_err),
 *   end_bias  [runs][6]  (nullable) gyro and accel bias estimates at n-1,
 *   consist   [runs][19] (nullable) over the GPS epochs >= stats_start, after the update: sums of the
 *             position / velocity / attitude block NEES [3], counts of |error_i| <= 3 sigma_i [15], epochs,
 *   dump_att/pos/vel/wb/ab (each nullable, all or none) [dump_runs][rows][3] histories.
 * ref_gyro, ref_accel [n][3], ref_nav [n][9] (att, pos LLA, vel NED), ref_gps [m][6],
 * gps_idx [m] (int64: IMU sample index of every GPS row, ascending), gps_vis [m]: DEVICE pointers. */
int b2ins_ins_loose_f64(const b2ins_ekf_config* cfg, const double* ref_gyro, const double* ref_accel,
                        const double* ref_nav, const double* ref_gps, const int64_t* gps_idx,
                        const double* gps_vis, double* end_err, double* end_bias, double* consist,
                        double* dump_att, double* dump_pos, double* dump_vel, double* dump_wb,
                        double* dump_ab, void* stream);

/* b2ins_ins_loose_f64 on vibrating sensors: every run's accelerometer and gyro samples carry the
 * vibration of vib_accel / vib_gyro (each nullable = none), added last, as b2ins_imu_noise_f64 adds it
 * (pathgen.py:477-493, :540-555): the filter sees the measurements K1 makes for the same runs.
 * VIB_SERIES: series [runs][3][series_len] on the device, for exactly the runs of this call (local run r
 * reads row r), e.g. from b2ins_psd_series_f64 with the same run_offset, ordered before this call on
 * `stream`.  The filter model itself knows nothing of the vibration (DESIGN.md section 11: raise vel_rw /
 * att_rw by sigma sqrt(dt) for random vibration).  b2ins_ins_loose_f64 is the NULL / NULL case. */
int b2ins_ins_loose_ex_f64(const b2ins_ekf_config* cfg, const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                           const double* ref_gyro, const double* ref_accel, const double* ref_nav,
                           const double* ref_gps, const int64_t* gps_idx, const double* gps_vis, double* end_err,
                           double* end_bias, double* consist, double* dump_att, double* dump_pos,
                           double* dump_vel, double* dump_wb, double* dump_ab, void* stream);

/* b2ins_ins_loose_ex_f64 that also reduces every run's process errors over the series: proc_stats
 * [runs][3][9] = max|e|, mean, std (ddof 0) of the attitude (wrapped to [-pi, pi]), position and velocity
 * errors of samples proc_start .. n-1 (proc_start in [0, n)), the reference's get_error_stats(err_stats_start
 * >= 0) (ins_data_manager.py:761-808).  Sample i's error is the state of history row i (after that sample's
 * GPS update) against ref_nav row i.  proc_pos_frame: the position columns, as in
 * b2ins_mc_free_integration_ex_f64 (B2INS_POS_FRAME_LLA differences, _NED or _ECEF metres).  Everything else,
 * including every other output, is b2ins_ins_loose_ex_f64's, bit for bit.  DEVICE pointers. */
int b2ins_ins_loose_proc_f64(const b2ins_ekf_config* cfg, const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                             int64_t proc_start, int proc_pos_frame, const double* ref_gyro, const double* ref_accel,
                             const double* ref_nav, const double* ref_gps, const int64_t* gps_idx,
                             const double* gps_vis, double* end_err, double* end_bias, double* consist,
                             double* proc_stats, double* dump_att, double* dump_pos, double* dump_vel,
                             double* dump_wb, double* dump_ab, void* stream);

/* K7 on SUPPLIED measurements (a drive log, another simulator, a saved experiment): the same filter,
 * reading every run's IMU and GPS samples instead of generating them.
 *   gyro, accel [runs][n][3] run-major (rad/s, m/s^2); gps [runs][m][6] LLA (rad, rad, m) and NED
 *   velocity (m/s), applied at IMU sample gps_idx[j] (int64, strictly ascending, in [0, n); shared by all
 *   runs) when gps_vis[j] > 0.
 * cfg: gyro_err, accel_err, gps_stdp / gps_stdv are the filter's model only (Q, R, P0); ini is the initial
 * state, plus the P0 draw of global run run_offset + r under seed when ini_draw is 1 (the draw of
 * b2ins_ins_loose_f64, so the generated experiment's measurements filter to its results); stats_start is
 * ignored: there is no consistency record (it needs the true biases).
 * ref_nav [n][9] and end_err [runs][9]: both or neither; end_bias, dump_*: as in b2ins_ins_loose_f64.
 * DEVICE pointers. */
int b2ins_ins_loose_fed_f64(const b2ins_ekf_config* cfg, int ini_draw, const double* gyro, const double* accel,
                            const double* gps, const int64_t* gps_idx, const double* gps_vis,
                            const double* ref_nav, double* end_err, double* end_bias, double* dump_att,
                            double* dump_pos, double* dump_vel, double* dump_wb, double* dump_ab, void* stream);

/* Alignment: the filter initialises itself from its measurements instead of starting at cfg->ini plus a P0
 * draw (DESIGN.md section 11, "Alignment"; demo_algorithms/ins_loose.py:54-126).  Roll and pitch come from the
 * mean of accelerometer samples 0..9 at sample 9; yaw is `yaw` (B2INS_ALIGN_YAW) or the course over ground
 * atan2(v_E, v_N) of the fix row's GPS velocity (B2INS_ALIGN_GPS).  The fix row is the latest visible GPS row
 * at or before sample 9, else the first visible row after it; the filter starts at s0 = max(9, its sample)
 * with position and velocity as measured there, the attitude propagated alone (no Earth or transport rate)
 * from sample 9, and a diagonal P0: stdp^2, stdv^2; level N / E (b^2 + b_drift^2 + vrw^2 fs / 10) / 9.80665^2
 * of accelerometer y / x; yaw yaw_var, or with B2INS_ALIGN_GPS (stdv_N^2 v_E^2 + stdv_E^2 v_N^2) / |v_h|^4;
 * plus arw^2 dt_gap + (b^2 + b_drift^2) dt_gap^2 of the gyro on the attitude; biases as without alignment.
 * History rows before the state exists are NaN (attitude before sample 9, position and velocity before s0;
 * wb, ab are 0), the consistency record takes the GPS epochs after s0, process statistics start at
 * max(proc_start, s0).  Without a visible GPS row at a sample < n (the host does not check: gps_idx and
 * gps_vis are device data) there is no fix: position and velocity stay NaN in every history row and in end_err,
 * the consistency record has no epochs, and proc_stats (max, mean and std) are NaN.  cfg->ini and cfg->ini_att_std[2]
 * are not used; no initial-state draw is made. */
#define B2INS_ALIGN_OFF 0
#define B2INS_ALIGN_YAW 1
#define B2INS_ALIGN_GPS 2
typedef struct {
  int32_t mode;         /* B2INS_ALIGN_* */
  int32_t reserved;
  double yaw;           /* B2INS_ALIGN_YAW: the heading [rad] */
  double yaw_var;       /* B2INS_ALIGN_YAW: its variance [rad^2], P0 of the yaw misalignment */
} b2ins_ekf_align;

/* b2ins_ins_loose_proc_f64 with alignment (align NULL or B2INS_ALIGN_OFF: b2ins_ins_loose_proc_f64 itself).
 * vib_gyro / vib_accel nullable; proc_start -1 with proc_stats NULL: no process statistics.  n >= 10.
 * DEVICE pointers. */
int b2ins_ins_loose_align_f64(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, const b2ins_vib* vib_gyro,
                              const b2ins_vib* vib_accel, int64_t proc_start, int proc_pos_frame,
                              const double* ref_gyro, const double* ref_accel, const double* ref_nav,
                              const double* ref_gps, const int64_t* gps_idx, const double* gps_vis, double* end_err,
                              double* end_bias, double* consist, double* proc_stats, double* dump_att,
                              double* dump_pos, double* dump_vel, double* dump_wb, double* dump_ab, void* stream);

/* b2ins_ins_loose_fed_f64 with alignment: the fix row's position and velocity are the supplied gps row; no
 * initial-state draw (align NULL or B2INS_ALIGN_OFF: b2ins_ins_loose_fed_f64 with ini_draw 0).  n >= 10.
 * DEVICE pointers. */
int b2ins_ins_loose_fed_align_f64(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, const double* gyro,
                                  const double* accel, const double* gps, const int64_t* gps_idx,
                                  const double* gps_vis, const double* ref_nav, double* end_err, double* end_bias,
                                  double* dump_att, double* dump_pos, double* dump_vel, double* dump_wb,
                                  double* dump_ab, void* stream);

/* Run-to-run turn-on bias (DESIGN.md sections 4 and 11): b2ins_ins_loose_align_f64 where every run also draws the
 * turn-on bias of gyro_run / accel_run (each nullable = none), b_run[c] = b[c] z0 of b2ins_run_err's pair j = c
 * (the draw b2ins_imu_noise_rx_f64 and b2ins_imu_run_err_f64 make for the same global run), added to the constant
 * bias cfg->*_err.b of the measurements.  The filter's model takes it into P0: the bias states start at
 * b_drift^2 + b^2 + b_std^2, the aligned level term at (b^2 + b_drift^2 + b_std^2 + vrw^2 fs / 10) / 9.80665^2 and
 * the gyro's growth over the gap at arw^2 dt_gap + (b^2 + b_drift^2 + b_std^2) dt_gap^2; Q is unchanged.  The
 * consistency record's true bias is b + b_run + the drift.  end_bias_err [runs][6] (nullable): the gyro then accel
 * bias estimates minus the true biases at sample n-1.  sf and ma must be zero (the filter has no states for them),
 * b finite and >= 0: B2INS_ERR_ARG before any CUDA call otherwise.  With no non-zero b and end_bias_err NULL this
 * is b2ins_ins_loose_align_f64, bit for bit.  DEVICE pointers. */
int b2ins_ins_loose_rx_f64(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, const b2ins_vib* vib_gyro,
                           const b2ins_vib* vib_accel, int64_t proc_start, int proc_pos_frame,
                           const double* ref_gyro, const double* ref_accel, const double* ref_nav,
                           const double* ref_gps, const int64_t* gps_idx, const double* gps_vis, double* end_err,
                           double* end_bias, double* consist, double* proc_stats, double* dump_att,
                           double* dump_pos, double* dump_vel, double* dump_wb, double* dump_ab,
                           const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, double* end_bias_err,
                           void* stream);

/* b2ins_ins_loose_fed_f64 (align NULL or B2INS_ALIGN_OFF) or b2ins_ins_loose_fed_align_f64 (ini_draw must then be
 * 0) whose model knows the turn-on bias of gyro_run / accel_run (each nullable): the supplied measurements carry
 * each run's bias, and only b enters the filter, in P0 as in b2ins_ins_loose_rx_f64.  Checks as there.  DEVICE
 * pointers. */
int b2ins_ins_loose_fed_rx_f64(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, int ini_draw,
                               const double* gyro, const double* accel, const double* gps, const int64_t* gps_idx,
                               const double* gps_vis, const double* ref_nav, double* end_err, double* end_bias,
                               double* dump_att, double* dump_pos, double* dump_vel, double* dump_wb, double* dump_ab,
                               const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, void* stream);

/* ---- housekeeping ------------------------------------------------------ */
int b2ins_version(void);
const char* b2ins_last_error(void);
int b2ins_device_count(void);
/* number of Allan cluster sizes allan.allan_var produces for (n, fs), allan.py:29-44;
 * fills m[0..] (may be NULL) -- host helper, no GPU */
int b2ins_allan_num_tau(int64_t n, double fs, int64_t* m, int m_cap);

/* ---- K2: strapdown free integration, noise supplied ---------------------
 * Replaces FreeIntegration.run + get_results (demo_algorithms/free_integration.py:63-180)
 * and the per-run dispatch loop InsAlgoMgr.run_algo (ins_algo_manager.py:73-95).
 * gyro [rad/s], accel [m/s^2]: `layout`; att [yaw,pitch,roll rad], pos (LLA rad,rad,m if
 * ref_frame 0, ECEF-offset xyz m if ref_frame 1), vel (NED m/s): same layout. */
int b2ins_free_integration_f64(int ref_frame, double fs, int64_t runs, int64_t n,
                               const double* gyro, const double* accel, int layout,
                               const double* ini, int ini_sets, int ini_rows,
                               int64_t run_offset, int earth_rot,
                               double* att, double* pos, double* vel,
                               int lanes_per_run, void* stream);
int b2ins_free_integration_f64_host(int ref_frame, double fs, int64_t runs, int64_t n,
                                    const double* gyro, const double* accel, int layout,
                                    const double* ini, int ini_sets, int ini_rows,
                                    int64_t run_offset, int earth_rot,
                                    double* att, double* pos, double* vel, int lanes_per_run);

/* The odometer variant with supplied data: FreeIntegration.run of
 * demo_algorithms/free_integration_odo.py:63-160.  odo: [R][n] (RUN_MAJOR) or [n][R]. */
int b2ins_free_integration_odo_f64(int ref_frame, double fs, int64_t runs, int64_t n,
                                   const double* gyro, const double* odo, int layout,
                                   const double* ini, int ini_sets, int ini_rows,
                                   int64_t run_offset, int earth_rot,
                                   double* att, double* pos, double* vel,
                                   int lanes_per_run, void* stream);

/* ---- K1: IMU sensor-error generator --------------------------------------
 * Replaces pathgen.acc_gen / gyro_gen / bias_drift (pathgen.py:441-594) for `runs` runs:
 * meas = ref + b + drift + white + vib with on-device Philox4x32-10 normals keyed by
 * (seed, run_offset + r).  ref_gyro / ref_accel: [n][3] shared true IMU output.
 * gyro / accel: outputs in `layout`.  z_dump (nullable): the 12 normals per (run, t) as
 * [R][n][12] = (acc_gm[3], acc_w[3], gyr_gm[3], gyr_w[3]) for injection into the
 * reference's np.random.randn call sequence.
 * A correlation time below dt / 2 gives a decay factor |a| = |1 - dt / b_corr| > 1: the drift grows as |a|^t
 * and, where the reference's serial recurrence overflows to alternating +-inf, the generators do not follow it
 * (measured at a = -3 and a = -1.5): this generator (and b2ins_imu_err_stats_f64) gives NaN once an infinity
 * enters a tile's scan, and for a = -1.5 +-inf; the fused Monte-Carlo kernels give alternating +-inf, a few
 * samples from where the reference overflows; b2ins_allan_mc_f64 gives NaN at every tau.  Inside the float64 range
 * all of them hold the drift to the same bound as for |a| <= 1. */
int b2ins_imu_noise_f64(double fs, int64_t runs, int64_t n,
                        const double* ref_gyro, const double* ref_accel,
                        const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                        const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                        uint64_t seed, int64_t run_offset, int layout,
                        double* gyro, double* accel, double* z_dump, void* stream);
int b2ins_imu_noise_f64_host(double fs, int64_t runs, int64_t n,
                             const double* ref_gyro, const double* ref_accel,
                             const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                             const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                             uint64_t seed, int64_t run_offset, int layout,
                             double* gyro, double* accel, double* z_dump);

/* K1 with the terms of b2ins_noise_terms added to every measurement (gyro_terms / accel_terms nullable: none).
 * Sensor 0 is accel, sensor 1 gyro; the walk of axis c draws pair 32 + 3 sensor + c (z0), the quantisation
 * uniform of sample t draw 38 + 3 sensor + c.  With every term zero these are b2ins_imu_noise_f64[_host]. */
int b2ins_imu_noise_ex_f64(double fs, int64_t runs, int64_t n,
                           const double* ref_gyro, const double* ref_accel,
                           const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                           const b2ins_noise_terms* gyro_terms, const b2ins_noise_terms* accel_terms,
                           const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                           uint64_t seed, int64_t run_offset, int layout,
                           double* gyro, double* accel, double* z_dump, void* stream);
int b2ins_imu_noise_ex_f64_host(double fs, int64_t runs, int64_t n,
                                const double* ref_gyro, const double* ref_accel,
                                const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                                const b2ins_noise_terms* gyro_terms, const b2ins_noise_terms* accel_terms,
                                const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                                uint64_t seed, int64_t run_offset, int layout,
                                double* gyro, double* accel, double* z_dump);

/* K1 with the IEEE Std 952 terms and the run-to-run errors of b2ins_run_err (gyro_run / accel_run nullable:
 * none).  With every run error zero these are b2ins_imu_noise_ex_f64[_host], which are this entry point with
 * null run errors. */
int b2ins_imu_noise_rx_f64(double fs, int64_t runs, int64_t n,
                           const double* ref_gyro, const double* ref_accel,
                           const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                           const b2ins_noise_terms* gyro_terms, const b2ins_noise_terms* accel_terms,
                           const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                           uint64_t seed, int64_t run_offset, int layout,
                           double* gyro, double* accel, double* z_dump,
                           const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, void* stream);
int b2ins_imu_noise_rx_f64_host(double fs, int64_t runs, int64_t n,
                                const double* ref_gyro, const double* ref_accel,
                                const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                                const b2ins_noise_terms* gyro_terms, const b2ins_noise_terms* accel_terms,
                                const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                                uint64_t seed, int64_t run_offset, int layout,
                                double* gyro, double* accel, double* z_dump,
                                const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run);
/* The run errors K1-rx and K9-rx draw for runs run_offset .. run_offset + runs - 1:
 * out [runs][2][12] (device; sensor 0 accel, 1 gyro): S row-major [9], then b_run [3].  Asynchronous. */
int b2ins_imu_run_err_f64(uint64_t seed, int64_t runs, int64_t run_offset, const b2ins_run_err* gyro_run,
                          const b2ins_run_err* accel_run, double* out, void* stream);

/* ---- K12: fused Monte-Carlo run (noise -> integration -> per-run errors) --
 * Replaces loop A (ins_sim.py:490-496) + loop B (ins_algo_manager.py:73-95) + the per-run
 * part of InsDataMgr.calc_data_err / array_error (ins_data_manager.py:454-541).
 *   ref_gyro, ref_accel [n][3]: true IMU output (pathgen.path_gen 'imu').
 *   ref_nav [n][9]: true att(yaw,pitch,roll), pos, vel per sample (pathgen 'nav',
 *            reordered).  Only row n-1 is read unless cfg->stats_start >= 0.
 *   ini [ini_sets][ini_rows].
 *   end_err [runs][9]: (att wrapped to [-pi,pi], pos, vel) error at sample n-1.
 *   end_state [runs][9] (nullable): att, pos, vel at sample n-1.
 *   proc_stats [runs][3][9] (nullable unless stats_start >= 0): per-run max|e|, mean, std
 *            (ddof 0) of the error over samples >= stats_start; positions as (lat, lon, alt) differences
 *            in ref_frame 0 (in metres: b2ins_mc_free_integration_ex_f64).
 *   dump_att/pos/vel, dump_gyro/accel (each nullable): [dump_runs][rows][3] histories, rows = n or
 *            ceil(n / cfg->dump_stride).
 * Asynchronous on `stream`. */
int b2ins_mc_free_integration_f64(const b2ins_mc_config* cfg,
                                  const double* ref_gyro, const double* ref_accel,
                                  const double* ref_nav, const double* ini,
                                  double* end_err, double* end_state, double* proc_stats,
                                  double* dump_att, double* dump_pos, double* dump_vel,
                                  double* dump_gyro, double* dump_accel, void* stream);
/* The same with the frame of the position columns of proc_stats (ref_frame 0 only; the attitude and
 * velocity columns and every other output are those of b2ins_mc_free_integration_f64):
 *   B2INS_POS_FRAME_LLA   (lat, lon, alt) differences -- b2ins_mc_free_integration_f64;
 *   B2INS_POS_FRAME_ECEF  metres, lla2ecef(x) - lla2ecef(truth) of every sample;
 *   B2INS_POS_FRAME_NED   metres, that difference rotated by ecef_to_ned of the true position of the sample
 * (array_error with extra_opt 'ned' / 'ecef', ins_data_manager.py:543-552).  NED and ECEF need
 * cfg->ref_frame == 0: ref_frame 1 positions are metres already. */
int b2ins_mc_free_integration_ex_f64(const b2ins_mc_config* cfg, int proc_pos_frame,
                                     const double* ref_gyro, const double* ref_accel,
                                     const double* ref_nav, const double* ini,
                                     double* end_err, double* end_state, double* proc_stats,
                                     double* dump_att, double* dump_pos, double* dump_vel,
                                     double* dump_gyro, double* dump_accel, void* stream);
/* Host-buffer convenience: copies ref/ini up, runs K12 + K3, copies end_err [runs][9] and
 * stats [3][9] back.  end_err may be NULL (stats only). */
int b2ins_mc_free_integration_f64_host(const b2ins_mc_config* cfg,
                                       const double* ref_gyro, const double* ref_accel,
                                       const double* ref_nav, const double* ini,
                                       double* end_err, double* stats);

/* ---- Monte-Carlo plan: the low-latency host path ----------------------------
 * A plan owns everything one experiment shape (n samples, up to `runs` runs, ini sets)
 * needs between calls: device buffers, pinned staging buffers and a stream.  plan_run is
 * b2ins_mc_free_integration_f64_host without the per-call allocations: stage the host
 * inputs into pinned memory, H2D copy (true IMU samples, ref_nav_end = the 9 values
 * att,pos,vel of the true trajectory at sample n-1, ini),
 * K12, K3, ONE D2H copy (stats [3][9] -- skipped with K3 if stats == NULL -- and, if end_err !=
 * NULL, the [runs][9] end-point errors), synchronise.  This is what Sim.run() calls on a single GPU.  A plan is bound to
 * the device current at creation and is not thread-safe (one plan per thread). */
typedef struct b2ins_mc_plan b2ins_mc_plan;
int b2ins_mc_plan_create(int64_t n, int64_t max_runs, int ini_sets, int ini_rows,
                         b2ins_mc_plan** plan);
int b2ins_mc_plan_run(b2ins_mc_plan* plan, const b2ins_mc_config* cfg,
                      const double* ref_gyro, const double* ref_accel, const double* ref_nav_end,
                      const double* ini, double* end_err, double* stats);
int b2ins_mc_plan_destroy(b2ins_mc_plan* plan);
/* Multi-GPU use: plan_run with stats == NULL skips K3 and only synchronises the end-point errors;
 * the DEVICE address of the plan's [max_runs][9] end_err buffer (valid until the next plan_run)
 * can then be handed to b2ins_error_stats_exchange_f64 on plan_stream(). */
double* b2ins_mc_plan_err_device(b2ins_mc_plan* plan);
void* b2ins_mc_plan_stream(b2ins_mc_plan* plan);

/* ---- K3: ensemble error statistics ---------------------------------------
 * Replaces InsDataMgr.__end_point_error_stats / __array_stats
 * (ins_data_manager.py:717-759, :797-808) on a [runs][ncomp] error matrix.
 * Two-phase so that a multi-GPU caller can all-reduce in between:
 *   phase 1: partial[0..ncomp) = sum e, partial[ncomp..2ncomp) = max|e|  (this shard)
 *   (caller all-reduces: SUM the first ncomp, MAX the second ncomp, and the run count)
 *   phase 2: given mean[ncomp], partial2[0..ncomp) = sum (e-mean)^2
 * b2ins_error_stats_f64 does both phases for a single shard and writes
 * stats [3][ncomp] = max|e|, mean, std(ddof 0).  ncomp <= 32.  All reductions are
 * deterministic (fixed order, no floating-point atomics).  workspace: device scratch of
 * b2ins_error_stats_workspace_bytes(ncomp) bytes.
 * Non-finite errors, here and in every max|e| / mean / std this library writes (K3x, K9, K3p,
 * K12 and K7 proc_stats), follow NumPy's np.max(np.abs(e)), np.average and np.std: a NaN in a
 * column makes its max, mean and std NaN; +-inf makes max inf, mean +-inf (NaN if both signs
 * occur) and std NaN.  The statistics of no samples are NaN.  K12 and K7 reduce in one pass
 * shifted by the first counted sample: if that sample is +-inf, its column reports max inf, mean
 * that infinity and std NaN whatever the later samples hold. */
int64_t b2ins_error_stats_workspace_bytes(int ncomp);
int b2ins_error_partial_f64(int64_t runs, int ncomp, const double* err, double* partial,
                            void* workspace, void* stream);
int b2ins_error_partial2_f64(int64_t runs, int ncomp, const double* err, const double* mean,
                             double* partial2, void* workspace, void* stream);
int b2ins_error_stats_f64(int64_t runs, int ncomp, const double* err, double* stats,
                          void* workspace, void* stream);

/* ---- K3x: statistics fused with their multi-GPU exchange ----------------------------------
 * One kernel per rank: shard statistics of err [runs][ncomp] (runs may be 0), peer stores of
 * (max, mean, std, count) into every rank's window over NVLink, flag exchange, Chan merge ->
 * stats [3][ncomp] of ALL ranks' runs on every rank.  No NCCL on the data path.
 *   windows[world]: DEVICE addresses, valid in THIS process, of each rank's receive window
 *       (rank's own included): 2 * world * 32 doubles of symmetric / peer-mapped memory, zeroed
 *       once before the first call;  seq: 1, 2, 3, ... per communicator (same on all ranks);
 *   every rank must make the same sequence of calls.  Needs runs * ncomp <= 2^17 per rank
 *   (the single-block path) and world <= 16.  timeout_flag: device int, set to 1 if a peer
 *   did not arrive within ~2 s. */
int b2ins_error_stats_exchange_f64(int64_t runs, int ncomp, const double* err, int rank, int world,
                                   const uint64_t* windows, uint64_t seq, double* stats,
                                   int* timeout_flag, void* stream);

/* ---- K4: Allan variance ---------------------------------------------------
 * Replaces allan.allan_var (allan/allan.py:18-59) for `nseries` series at once.
 * Series s, sample t lives at x[s / inner * outer_stride + (s % inner) + t * sample_stride]
 * (RUN_MAJOR accel [R][n][3]: inner = 3, outer_stride = 3n, sample_stride = 3).
 * inner >= 1, sample_stride >= 1 and outer_stride >= 0, else B2INS_ERR_ARG (as for K4o and K11).
 * avar [nseries][ntau], tau [ntau], ntau = b2ins_allan_num_tau(n, fs).
 * workspace: device scratch of b2ins_allan_workspace_bytes(n, nseries) bytes. */
int64_t b2ins_allan_workspace_bytes(int64_t n, int64_t nseries);
int b2ins_allan_f64(double fs, int64_t n, int64_t nseries, const double* x,
                    int64_t inner, int64_t outer_stride, int64_t sample_stride,
                    double* avar, double* tau, void* workspace, void* stream);
int b2ins_allan_f64_host(double fs, int64_t n, int64_t nseries, const double* x,
                         int64_t inner, int64_t outer_stride, int64_t sample_stride,
                         double* avar, double* tau);

/* ---- K4o: overlapping Allan variance ---------------------------------------
 * avar_o(m) = 1 / (2 m^2 M) sum_{k<M} (S(k+m, m) - S(k, m))^2, S(k, m) = x_k + ... + x_{k+m-1},
 * M = n - 2m + 1 (NIST SP 1065 eq. 10): every start offset k, on the cluster sizes m of K4's grid
 * (ntau = b2ins_allan_num_tau(n, fs), the same tau).  Series addressing as b2ins_allan_f64.
 * A series with a NaN sample gives NaN at every tau; one with +-inf samples gives what the
 * definitional sum gives in IEEE arithmetic (+inf, or NaN where a window holds inf - inf).
 * avar [nseries][ntau], tau [ntau]; workspace: b2ins_oallan_workspace_bytes(n, nseries) bytes
 * (about 16 B per series-sample).  Deterministic: bit-identical whatever the batch. */
int64_t b2ins_oallan_workspace_bytes(int64_t n, int64_t nseries);
int b2ins_oallan_f64(double fs, int64_t n, int64_t nseries, const double* x,
                     int64_t inner, int64_t outer_stride, int64_t sample_stride,
                     double* avar, double* tau, void* workspace, void* stream);
int b2ins_oallan_f64_host(double fs, int64_t n, int64_t nseries, const double* x,
                          int64_t inner, int64_t outer_stride, int64_t sample_stride,
                          double* avar, double* tau);

/* ---- K4o, Hadamard form: overlapping Hadamard variance -------------------------
 * hvar(m) = 1 / (6 m^2 H) sum_{k<H} (S(k+2m, m) - 2 S(k+m, m) + S(k, m))^2, H = n - 3m + 1
 * (NIST SP 1065), on the same cluster sizes and tau as b2ins_oallan_f64: a second difference of
 * adjacent window sums, so a linear drift of the samples cancels, and white noise gives sigma^2 / m.
 * Signature, series addressing, outputs and workspace (b2ins_oallan_workspace_bytes) as
 * b2ins_oallan_f64.  A series with a NaN sample gives NaN at every tau; one with +-inf samples gives
 * what the definitional sum gives in IEEE arithmetic: NaN where a term's contributions +S(k+2m),
 * -2 S(k+m), +S(k) hold both infinities, else +inf.  Deterministic: bit-identical whatever the batch. */
int b2ins_ohadamard_f64(double fs, int64_t n, int64_t nseries, const double* x,
                        int64_t inner, int64_t outer_stride, int64_t sample_stride,
                        double* hvar, double* tau, void* workspace, void* stream);
int b2ins_ohadamard_f64_host(double fs, int64_t n, int64_t nseries, const double* x,
                             int64_t inner, int64_t outer_stride, int64_t sample_stride,
                             double* hvar, double* tau);

/* ---- K13: Allan noise identification (IEEE Std 952-1997 Annex C) ----------------------
 * Fits sigma^2(tau) = C_-2 tau^-2 + C_-1 tau^-1 + C_0 + C_1 tau + C_2 tau^2 (every C_p >= 0) to the Allan
 * variance curves of `nseries` series of n samples at fs, as K4 or K4o computed them (the variance, not the
 * deviation), on their grid: tau_k = m_k / fs with m_k from b2ins_allan_num_tau(n, fs), weights
 * w_k = floor(n / m_k) - 1.  Objective sum_k w_k (model(tau_k) / v_k - 1)^2 over the bins with v_k > 0, minimised
 * exactly over the non-negative coefficients by enumerating the 31 supports (DESIGN.md section 3.13).
 * var: v of series s, bin k at var[s * series_stride + k * bin_stride] (device; K4's [nseries][ntau] is
 * series_stride = ntau, bin_stride = 1; may be null when ntau = 0).  out [nseries][6] (device):
 *   Q = sqrt(C_-2 / 3), N = sqrt(C_-1), B = sqrt(C_0 pi / (2 ln 2)), K = sqrt(3 C_1), R = sqrt(2 C_2),
 *   B_min = sqrt(min_k v_k) / sqrt(2 ln 2 / pi).
 * A NaN, +-inf or negative v_k, or ntau = 0, gives six NaNs; a zero bin is left out of the fit but counts for
 * B_min; all-zero bins give six zeros.  fs > 0 and finite, n >= 0, nseries >= 0, series_stride >= 0 and
 * bin_stride >= 1, else B2INS_ERR_ARG; nseries = 0 returns B2INS_OK.  Deterministic: a series gives the same
 * bits whatever the batch and its position in it. */
int b2ins_allan_fit_f64(double fs, int64_t n, int64_t nseries, const double* var, int64_t series_stride,
                        int64_t bin_stride, double* out, void* stream);
int b2ins_allan_fit_f64_host(double fs, int64_t n, int64_t nseries, const double* var, int64_t series_stride,
                             int64_t bin_stride, double* out);

/* ---- K5: vibration series from a PSD -------------------------------------------
 * Replaces time_series_from_psd (gnss_ins_sim/psd/time_series_from_psd.py:17-65) as called
 * three times per sensor and run by acc_gen / gyro_gen (pathgen.py:478-485, :541-548).
 * freq [table_len], sxx3 [3][table_len] (x, y, z single-sided PSD): DEVICE pointers, already
 * cut at fs/2 like Sim.__parse_env does (ins_sim.py:688-697).  sensor: 0 accel, 1 gyro (selects
 * the Philox draw ids of the random phases).  series [runs][3][N], N = b2ins_psd_series_len(n);
 * hand it to b2ins_vib.series with series_len = N (the consumer tiles it to n samples).
 * workspace: b2ins_psd_workspace_bytes(n, runs) bytes of device scratch. */
int b2ins_psd_series_len(int64_t n);
int64_t b2ins_psd_workspace_bytes(int64_t n, int64_t runs);
int b2ins_psd_series_f64(double fs, int64_t n, int64_t runs, int sensor, int table_len,
                         const double* freq, const double* sxx3, uint64_t seed,
                         int64_t run_offset, double* series, void* workspace, void* stream);

/* ---- K11: Welch power spectral density ---------------------------------------------
 * scipy.signal.welch(x, fs, window, nperseg, noverlap) with detrend='constant', scaling='density',
 * average='mean', one-sided, nfft = nperseg, for `nseries` series at once.  N = nperseg, D = noverlap,
 * S = N - D, K = (n - D) / S segments (samples after the last are unused), L = N / 2 + 1:
 *   psd[k] = (1/K) sum_j c_k |DFT_N((x_j - mean x_j) w)[k]|^2 / (fs sum w^2), c_0 = c_{L-1} = 1, else 2;
 *   freq[k] = k / (N (1/fs)), as np.fft.rfftfreq.
 * N must be even, >= 16, and a power of two up to 16384 or at most 8192; 0 <= D < N; n >= N.
 * Series addressing as b2ins_allan_f64.  window [N] (device): any finite window.  psd [nseries][L],
 * freq [L] (device).  A NaN or +-inf sample inside a used segment makes every bin of its series NaN.
 * Deterministic: a series gives the same bits whatever the batch, its position and its layout.
 * b2ins_welch_workspace_bytes: device scratch for these arguments, negative if nperseg is not a
 * length this transform takes (or noverlap, n do not give a segment). */
int64_t b2ins_welch_workspace_bytes(int64_t n, int64_t nseries, int64_t nperseg, int64_t noverlap);
int b2ins_welch_f64(double fs, int64_t n, int64_t nseries, const double* x,
                    int64_t inner, int64_t outer_stride, int64_t sample_stride,
                    int64_t nperseg, int64_t noverlap, const double* window,
                    double* psd, double* freq, void* workspace, void* stream);
int b2ins_welch_f64_host(double fs, int64_t n, int64_t nseries, const double* x,
                         int64_t inner, int64_t outer_stride, int64_t sample_stride,
                         int64_t nperseg, int64_t noverlap, const double* window,
                         double* psd, double* freq);

/* ---- K6: GPS measurement generator ---------------------------------------------------
 * Replaces pathgen.gps_gen (gnss_ins_sim/pathgen/pathgen.py:596-625) and its call in loop A
 * (gnss_ins_sim/sim/ins_sim.py:497-500) for `runs` runs at once:
 *   gps[r][k] = ref_gps[k] + (pos_err, stdv) * N(0,1),   Philox draws (k, 24..26, run_offset + r).
 * ref_gps [m][6] (device): position (LLA rad/rad/m if gps_type 0 = ref_frame 0, xyz m if 1) and
 * NED velocity, as path_gen's 'gps' columns 1..6.  stdp / stdv: host [3], metres and m/s; with
 * gps_type 0 the horizontal position sigmas are converted to radians at ref_gps[0], like the
 * reference.  gps [runs][m][6] (device). */
int b2ins_gps_noise_f64(int64_t runs, int64_t m, const double* ref_gps, const double* stdp,
                        const double* stdv, int gps_type, uint64_t seed, int64_t run_offset,
                        double* gps, void* stream);

/* ---- K8: magnetometer measurement generator ------------------------------------------
 * Replaces pathgen.mag_gen (gnss_ins_sim/pathgen/pathgen.py:643-661) and its call in loop A
 * (gnss_ins_sim/sim/ins_sim.py:501-503) for `runs` runs at once, at the IMU rate:
 *   mag[r][k] = si (ref_mag[k] + hi) + std * N(0,1),
 * Philox draws (k, 13, run_offset + r) -> (x, y) and z0 of (k, 14, run_offset + r) -> z.
 * ref_mag [n][3] (device): true field in the body frame [uT], path_gen's 'mag' columns 1..3.
 * si: host [9], soft-iron matrix, row-major; hi, std: host [3], hard iron and noise sigma [uT]
 * (std finite and >= 0).  mag [runs][n][3] (device), run-major. */
int b2ins_mag_noise_f64(int64_t runs, int64_t n, const double* ref_mag, const double* si,
                        const double* hi, const double* std, uint64_t seed, int64_t run_offset,
                        double* mag, void* stream);

/* ---- K10: soft- and hard-iron magnetometer calibration -------------------------------
 * MagCalibrate (demo_algorithms/mag_calibrate_src/src/MagCalibration.c:34-306) for `runs` runs at once,
 * one CTA per run (DESIGN.md section 3.11).  seg: host [6] = (x0, xf, y0, yf, z0, zf), half-open sample
 * ranges of the rotations about the sensor's x, y and z axes, each >= 3 rows inside [0, n).
 * Outputs (device): soft_iron [runs][9] (row-major S) and hard_iron [runs][4] (hard iron, field radius);
 * calibrated samples are S m - hard_iron[0:3].  A singular 3x3 or 4x4 system, or any non-finite output (a
 * NaN or +-inf sample, a zero range, moments past the range of double), gives NaN in all 13 values of the run
 * and in its mag_cal rows.  The result scales with the samples' units bit for bit.  Deterministic: a run's
 * result is bit-identical whatever runs, run_offset or the other runs.
 * b2ins_magcal_f64: the samples of K8 (b2ins_mag_noise_f64 with the same ref_mag, si, hi, std, seed and
 *   run_offset), regenerated, never stored.  err [runs][13] (nullable): the calibration error against that
 *   model, with k = trace(S si) / 3: S si / k - I (9), hard_iron[0:3] / k - hi (3), hard_iron[3] / k - |ref_mag[0]|.
 * b2ins_magcal_fed_f64: sample k of run r at mag[r * run_stride + k * sample_stride + c] (device;
 *   sample_stride >= 3).  mag_cal [runs][L][3] (nullable), L = the three lengths summed: the segments stacked,
 *   after the reference's staged corrections O m, diag(s) ., - hard_iron[0:3].
 * b2ins_magcal_fed_f64_host: the fed form on host buffers (synchronous). */
int b2ins_magcal_f64(int64_t runs, int64_t n, const int64_t* seg, const double* ref_mag, const double* si,
                     const double* hi, const double* std, uint64_t seed, int64_t run_offset, double* soft_iron,
                     double* hard_iron, double* err, void* stream);
int b2ins_magcal_fed_f64(int64_t runs, int64_t n, const int64_t* seg, const double* mag, int64_t run_stride,
                         int64_t sample_stride, double* soft_iron, double* hard_iron, double* mag_cal,
                         void* stream);
int b2ins_magcal_fed_f64_host(int64_t runs, int64_t n, const int64_t* seg, const double* mag, int64_t run_stride,
                              int64_t sample_stride, double* soft_iron, double* hard_iron, double* mag_cal);

/* ---- K9: IMU error statistics, reduced inside the noise generator ---------------------
 * InsDataMgr.get_error_stats('gyro' | 'accel') (ins_data_manager.py:385-452, :524-541, :717-808) for
 * `runs` runs without materialising them: the measurements of b2ins_imu_noise_f64 (same arguments, same
 * Philox draws, the same values) minus the truth, e = meas - ref, reduced per run.
 *   end_err [runs][6] (device): e at sample n-1; columns accel x, y, z, then gyro x, y, z.
 *   proc_stats [runs][3][6] (device; may be NULL when stats_start < 0): max|e|, mean and std (ddof 0)
 *       over samples >= stats_start, same columns.
 * stats_start < 0: end_err only; otherwise stats_start < n.  Deterministic (fixed-order reductions, no
 * floating-point atomics).  Asynchronous on `stream`. */
int b2ins_imu_err_stats_f64(double fs, int64_t runs, int64_t n,
                            const double* ref_gyro, const double* ref_accel,
                            const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                            const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                            uint64_t seed, int64_t run_offset, int64_t stats_start,
                            double* end_err, double* proc_stats, void* stream);
/* K9 of the measurements b2ins_imu_noise_ex_f64 makes (same arguments); with every term zero, K9 itself. */
int b2ins_imu_err_stats_ex_f64(double fs, int64_t runs, int64_t n,
                               const double* ref_gyro, const double* ref_accel,
                               const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                               const b2ins_noise_terms* gyro_terms, const b2ins_noise_terms* accel_terms,
                               const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                               uint64_t seed, int64_t run_offset, int64_t stats_start,
                               double* end_err, double* proc_stats, void* stream);
/* K9 of the measurements b2ins_imu_noise_rx_f64 makes (the _ex arguments plus the nullable run errors); with
 * null or all-zero run errors, b2ins_imu_err_stats_ex_f64. */
int b2ins_imu_err_stats_rx_f64(double fs, int64_t runs, int64_t n,
                               const double* ref_gyro, const double* ref_accel,
                               const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                               const b2ins_noise_terms* gyro_terms, const b2ins_noise_terms* accel_terms,
                               const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                               uint64_t seed, int64_t run_offset, int64_t stats_start,
                               double* end_err, double* proc_stats,
                               const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, void* stream);

/* ---- K3p: per-run error statistics of a device array ----------------------------------
 * x [runs][m][ncomp] against the shared ref [m][ncomp] (device), e = x - ref:
 *   end_err [runs][ncomp]: e at row m-1;
 *   proc_stats [runs][3][ncomp]: max|e|, mean and std (ddof 0) over rows >= start (0 <= start < m).
 * 1 <= ncomp <= 8.  Deterministic.  Asynchronous on `stream`. */
int b2ins_proc_stats_f64(int64_t runs, int64_t m, int ncomp, const double* x, const double* ref,
                         int64_t start, double* end_err, double* proc_stats, void* stream);

/* ---- host: true-trajectory generator -----------------------------------------------
 * Replaces pathgen.path_gen (gnss_ins_sim/pathgen/pathgen.py:26-329, with
 * calc_true_sensor_output :331-411 and parse_motion_def :413-439).  Plain CPU code (the
 * trajectory is generated once, serially in time, and shared by all runs); no GPU needed.
 *   ini [9]: lat, lon [rad], alt, body velocity, yaw, pitch, roll [rad];
 *   motion_def [segs][9]: type, 3 attitude commands [rad | rad/s], 3 velocity commands, duration
 *       [s], gps visibility -- as Sim.__parse_motion produces them (ins_sim.py:578-610);
 *   mobility [3]: max acceleration, max angular acceleration [rad/s^2], max angular rate [rad/s];
 *   fs: IMU rate; osr: simulation over-sampling ratio (1); fs_gps, fs_odo: only used if the
 *       matching output buffer is given.
 *   imu [cap][7] (index, accel xyz, gyro xyz), nav [cap][10] (index, pos, vel NED, yaw pitch roll),
 *   gps [cap][8] (nullable), odo [cap][5] (nullable).  cap >= b2ins_path_rows(...).
 * Returns the number of imu/nav rows written, or < 0: -2 negative duration, -3 empty, -4 cap too
 * small, -5 unknown command type.  b2ins_path_gen_host generates no magnetometer output; it is
 * b2ins_path_gen_ex_host with a null geomag_n.
 * b2ins_path_gen_ex_host: geomag_n [3] (nullable) is the geomagnetic field in the navigation frame
 *   [uT] (WMM at the initial position, pathgen.py:164-171; gnss_ins_sim_b200/geomag.py evaluates
 *   it); with it, mag [cap][4] gets (index, c_nb^T geomag_n) on every imu/nav row. */
int64_t b2ins_path_rows(const double* motion_def, int64_t segs, double fs);
int64_t b2ins_path_gen_host(const double* ini, const double* motion_def, int64_t segs, double fs,
                            double osr, double fs_gps, double fs_odo, const double* mobility,
                            int ref_frame, int64_t cap, double* imu, double* nav, double* gps,
                            int64_t* gps_rows, double* odo);
int64_t b2ins_path_gen_ex_host(const double* ini, const double* motion_def, int64_t segs, double fs,
                               double osr, double fs_gps, double fs_odo, const double* mobility,
                               int ref_frame, int64_t cap, double* imu, double* nav, double* gps,
                               int64_t* gps_rows, double* odo, const double* geomag_n, double* mag);

/* ---- diagnostics ---------------------------------------------------------
 * Measured FP64 FMA issue rate of the current device [lane-FMA/s]: a ~10 ms dependent-chain
 * microbenchmark (8 independent chains per thread, every SM filled).  The Monte-Carlo
 * kernels are FP64-instruction-bound, so this is the denominator bench.py reports their
 * FP64 utilisation against (beside the HBM roofline).  Synchronous. */
int b2ins_diag_dfma_rate(double* dfma_per_s);

/* The lanes-per-run value lanes_per_run = 0 resolves to, for `runs` runs on `sm_count` SMs
 * (0: the current device, 132 if there is none).  fused: the launch is the fused Monte-Carlo kernel
 * with end-point statistics only (the warp-specialised form applies); otherwise supplied data or
 * process statistics.  A pure function of its arguments: usable without a GPU. */
int b2ins_diag_auto_lanes(int64_t runs, int fused, int sm_count);

/* The launch shape of the fused, warp-specialised Monte-Carlo kernel for a lane-group width and a
 * reference frame: shape3[0] = producer warps per integrator warp (per channel for the split form),
 * [1] = integrator warps per CTA (2: the step split over an attitude and a velocity warp, ref_frame 1),
 * [2] = 1 if the lanes of a group share the trigonometry of a step (0 for the single-warp form: all zero).
 * Honours the tools' B2INS_MC_SHAPE override, i.e. reports what a launch would use.  Pure host logic. */
int b2ins_diag_mc_shape(int lanes_per_run, int ref_frame, int* shape3);

/* The transform b2ins_psd_series_f64 uses for a series of n samples (N = b2ins_psd_series_len(n),
 * M = N / 2): returns 0 for the direct cosine synthesis, 1 for the radix-2 transform of length M
 * (M a power of two) and 2 for Bluestein, and writes the transform length to *P (M, the Bluestein
 * length, or 0 for the direct synthesis).  Honours the tools' B2INS_PSD_DIRECT override (read once
 * per process, as the launch reads it).  Returns -1 if n <= 0 or P is NULL.  Pure host logic. */
int b2ins_diag_psd_plan(int64_t n, int* P);

/* The Gauss-Markov coefficients and the time segmentation b2ins_imu_noise_f64 and b2ins_imu_err_stats_f64
 * use for `runs` runs of n samples on `sm_count` SMs (0: the current device, 132 if there is none):
 * coef [3][6] = (gm_a, gm_b, wd) of the channels accel x y z, gyro x y z, as digested from the error models
 * (d[t+1] = gm_a d[t] + gm_b z0[t], plus wd z0[t] for b_corr = +inf); plan [3] = (nseg, seg_len, pass1_len):
 * nseg time segments of seg_len samples (the last one shorter), pass 1 reducing the last pass1_len samples
 * of each (0 for nseg = 1).  Pass 1 is shortened only where every channel's |gm_a|^pass1_len < 1e-20.
 * Pure host logic: the function the launch calls. */
int b2ins_diag_noise_plan(double fs, int64_t runs, int64_t n, const b2ins_sensor_err* gyro_err,
                          const b2ins_sensor_err* accel_err, int sm_count, double* coef, int64_t* plan);
/* The plan of the _ex entry points: as above; a non-zero rate random walk (k) never decays, so pass 1 then
 * covers whole segments (pass1_len = seg_len). */
int b2ins_diag_noise_plan_ex(double fs, int64_t runs, int64_t n, const b2ins_sensor_err* gyro_err,
                             const b2ins_sensor_err* accel_err, const b2ins_noise_terms* gyro_terms,
                             const b2ins_noise_terms* accel_terms, int sm_count, double* coef, int64_t* plan);

/* The device's own FP64 primitives (csrc/fastmath64.cuh, and mech.cuh's sincos_angle), applied
 * elementwise to n arguments: out0[i] = f(a[i]) (div: a[i] / b[i]); the sin/cos functions write
 * sin to out0 and cos to out1.  Each kernel inlines the production function itself.  Device
 * pointers; synchronous.  An unknown fn is B2INS_ERR_ARG. */
enum {
  B2INS_FM_RCP = 0,          /* rcp_nr(a)           */
  B2INS_FM_DIV = 1,          /* div_nr(a, b)        */
  B2INS_FM_SQRT = 2,         /* sqrt_nr(a)          */
  B2INS_FM_RSQRT = 3,        /* rsqrt_nr(a)         */
  B2INS_FM_SINCOS = 4,       /* sincos_bounded(a)   */
  B2INS_FM_SINCOS_ANGLE = 5, /* sincos_angle(a)     */
  B2INS_FM_SINCOSPI = 6,     /* sincospi_2u(a)      */
  B2INS_FM_LOG = 7           /* log_unit(a)         */
};
int b2ins_diag_fastmath_f64(int fn, int64_t n, const double* a, const double* b, double* out0, double* out1);

/* The noise generator's Philox4x32-10 on n (counter[4], key[2]) rows of ctr_key [n][6]:
 * words [n][4].  Device pointers; synchronous. */
int b2ins_diag_philox(int64_t n, const uint32_t* ctr_key, uint32_t* words);

/* The noise generator's Box-Muller pair from n Philox outputs words [n][4] (the normal_from_words
 * that every noise draw goes through): z [n][2] = (z0, z1).  Device pointers; synchronous. */
int b2ins_diag_normal_from_words(int64_t n, const uint32_t* words, double* z);

#ifdef __cplusplus
}
#endif
#endif /* B2INS_H_ */
