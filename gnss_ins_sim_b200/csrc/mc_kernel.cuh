// K2 / K12: the Monte-Carlo strapdown kernel.
//
// One LANE GROUP of G lanes (G = 1,2,4,...,32) owns one Monte-Carlo run; G = 32 is
// "one warp owns one run".  Per block of G consecutive samples:
//   phase A (time-parallel): lane j prepares sample base+j -- Philox4x32-10 + Box-Muller
//           normals, white noise, constant bias, vibration added to the true IMU sample
//           (read from the TMA-staged shared-memory tile), or the fed gyro/accel sample.
//   phase B (serial in time): for k = 0..G-1 every lane of the group pulls sample base+k
//           from lane k by warp shuffle, advances the Gauss-Markov bias and the 9-DoF
//           strapdown state (registers, replicated across the group) by one step.
// The shared true trajectory (ref gyro/accel [n][3], optionally ref nav [n][9]) is staged
// through shared memory in tiles of kTile samples by 1-D bulk async copies (TMA) completing
// on mbarriers, kStages deep, one pipeline per CTA shared by all its runs.
#pragma once
#include "mech.cuh"

namespace b2ins {

// Optional phase clocks (tools only: -DB2INS_PHASE_CLOCKS builds libb2ins_prof.so).  Slots 0-7:
// mc_kernel / mc_spec_kernel, 8-15: mc_av_kernel (see there).
constexpr int kPhaseClocks = 16;
#ifdef B2INS_PHASE_CLOCKS
__device__ unsigned long long g_phase_clocks[kPhaseClocks];
#define B2_CLK(var) const long long var = clock64()
#define B2_ACC(i, t0, t1) \
  if ((threadIdx.x & 31) == 0) atomicAdd(&g_phase_clocks[i], static_cast<unsigned long long>((t1) - (t0)))
#else
#define B2_CLK(var)
#define B2_ACC(i, t0, t1)
#endif

constexpr int kWarps = 4;
constexpr int kThreads = kWarps * 32;
constexpr int kTile = 128;   // samples per shared-memory tile (multiple of 32)
constexpr int kStagesFast = 3;   // pipeline depth; 2 when the 72 B/sample nav tile is staged too
template <bool PROC>
struct Stages {
  static constexpr int value = PROC ? 2 : kStagesFast;
};

// error model of one triad, pre-digested on the host (bias_drift: pathgen.py:583-586)
struct TriadNoise {
  double b[3];        // constant bias
  double gm_a[3];     // 1 - dt/tau            (0 if the drift is white)
  double gm_b[3];     // drift*sqrt(1-exp(-2dt/tau))  (0 if the drift is white)
  double wd[3];       // drift sigma if the drift is white (corr = inf), else 0
  double w[3];        // rw / sqrt(dt)
  int vib_type;
  int series_len;
  double vib_amp[3];
  double vib_w;       // ((2 pi) f) dt
  const double* series;  // [runs][3][series_len]
};

struct McParams {
  int64_t n, runs, run_offset, ini_offset;
  double dt;
  int earth_rot;
  uint32_t k0, k1;
  TriadNoise gyro, accel;
  const double* ref_gyro;   // [n][3]
  const double* ref_accel;  // [n][3]
  const double* ref_nav;    // [n][9] att, pos, vel
  const double* ini;        // [ini_sets][ini_rows]
  int ini_sets, ini_rows;
  // fed measurements (K2) -- element (r,t,c) at r*sr + t*st + c*sc
  const double* fed_gyro;
  const double* fed_accel;
  int64_t sr, st, sc;
  // odometer variant (free_integration_odo): algo = 1
  int algo;
  const double* ref_odo;   // [n] true forward speed (pathgen 'odo')
  double odo_scale, odo_stdv;
  const double* fed_odo;   // K2: element (r,t) at r*so_r + t*so_t
  int64_t so_r, so_t;
  // histories for runs [0, dump_runs): same stride convention
  double* out_att;
  double* out_pos;
  double* out_vel;
  double* out_gyro;
  double* out_accel;
  double* out_odo;     // [dump_runs][n] (algo 1)
  double* out_quat;    // [dump_runs][rows][4] scalar-first quaternion of every kept attitude sample
  int64_t osr, ost, osc;
  int64_t dump_runs;
  int64_t dump_stride; // >= 1: histories keep samples 0, s, 2s, ... (rows = ceil(n / s))
  int64_t dump_rows;
  // per-run results
  double* end_err;     // [runs][9]
  double* end_state;   // [runs][9]
  double* proc_stats;  // [runs][3][9]
  int64_t stats_start;
  int debug;           // tools (B2INS_PHASE_CLOCKS builds only): 1 = producers idle, 2 = integrators (A in
                       // mc_av_kernel) idle, 4 = V idle (mc_av_kernel)
  int proc_pos_frame;  // ref_frame 0 position columns of proc_stats: 0 LLA, 1 NED metres, 2 ECEF metres
};

// Prepared samples of one block, one slot per lane: phase A stores (gyro xyz, accel xyz),
// phase B reads sample k of its group with three 128-bit broadcast loads instead of twelve
// 32-bit shuffles.  48 B per lane; row padding keeps the group bases on distinct banks.
struct alignas(16) SampleSlot {
  double g[3], a[3];
};

template <bool PROC>
struct TileSmem {
  static constexpr int kStages = Stages<PROC>::value;
  alignas(128) double gyro[kStages][kTile * 3];
  alignas(128) double accel[kStages][kTile * 3];
  alignas(128) double nav[kStages][PROC ? kTile * 9 : 2];  // only staged for process statistics
  alignas(16) SampleSlot slot[kWarps][32];
  alignas(8) uint64_t full[kStages];
  alignas(8) uint64_t empty[kStages];
};

// Issue the copies of one tile: the 16-byte-multiple part by bulk async copy (TMA)
// completing on full[s]; an odd sample count leaves one 8-byte tail copied by hand.
// Smem: TileSmem, or the warp-specialised kernels' layouts (gyro and accel only: FED = PROC = false).
template <bool FED, bool PROC, class Smem>
__device__ __forceinline__ void issue_tile(Smem& sm, const McParams& p, int64_t tile, int s) {
  const int64_t t0 = tile * kTile;
  const uint32_t cnt = static_cast<uint32_t>(min64(kTile, p.n - t0));
  uint32_t tx = 0;
  if (!FED) tx += 2u * ((cnt * 24u) & ~15u);
  if (PROC) tx += (cnt * 72u) & ~15u;
  // the hand-copied tails are ordered before the arrive (release) below
  if constexpr (!FED) {
    if ((cnt * 24u) & 8u) {
      const uint32_t o = ((cnt * 24u) & ~15u) / 8;
      sm.gyro[s][o] = p.ref_gyro[t0 * 3 + o];
      sm.accel[s][o] = p.ref_accel[t0 * 3 + o];
    }
  }
  if constexpr (PROC) {
    if ((cnt * 72u) & 8u) {
      const uint32_t o = ((cnt * 72u) & ~15u) / 8;
      sm.nav[s][o] = p.ref_nav[t0 * 9 + o];
    }
  }
  mbar_arrive_expect_tx(&sm.full[s], tx);
  if constexpr (!FED) {
    const uint32_t b = (cnt * 24u) & ~15u;
    if (b) {
      bulk_g2s(sm.gyro[s], p.ref_gyro + t0 * 3, b, &sm.full[s]);
      bulk_g2s(sm.accel[s], p.ref_accel + t0 * 3, b, &sm.full[s]);
    }
  }
  if constexpr (PROC) {
    const uint32_t b = (cnt * 72u) & ~15u;
    if (b) bulk_g2s(sm.nav[s], p.ref_nav + t0 * 9, b, &sm.full[s]);
  }
}

// Refill the stage the PREVIOUS tile used (its consumers have had a whole tile to release it, so the
// issuing thread hardly ever waits), then wait for tile `tile`'s data in stage s, phase `parity`.
// 32-bit counts: n < 2^32 (b2ins_api.cu).  Phase clock slot `clk` times the wait.
template <bool FED, bool PROC, class Smem>
__device__ __forceinline__ void refill_and_wait(Smem& sm, const McParams& p, bool issuer, int tile,
                                                int num_tiles, int s, uint32_t parity, int clk) {
  constexpr int kStages = sizeof(Smem::full) / sizeof(uint64_t);
  if (issuer && tile >= 1 && tile - 1 + kStages < num_tiles) {
    const int sp = (tile - 1) % kStages;
    mbar_wait(&sm.empty[sp], static_cast<uint32_t>(((tile - 1) / kStages) & 1));
    issue_tile<FED, PROC>(sm, p, tile - 1 + kStages, sp);
  }
  B2_CLK(cw0);
  mbar_wait(&sm.full[s], parity);
  B2_CLK(cw1);
  B2_ACC(clk, cw0, cw1);
}

// Vibration term of one axis (pathgen.py:477-493 / :540-555); only called when a model is on.
__device__ __forceinline__ double vib_term(const TriadNoise& e, int c, int sensor, uint32_t t,
                                           uint32_t run_lo, uint32_t run_hi, uint32_t k0,
                                           uint32_t k1, int64_t run_local, const double* phase) {
  if (e.vib_type == 1) {
    const Normal2 zv = normal_pair(t, kDrawVib + c, run_lo, run_hi, k0, k1);
    return e.vib_amp[c] * (sensor == 0 ? zv.z0 : zv.z1);
  }
  if (e.vib_type == 2) {
    const double arg = e.vib_w * static_cast<double>(t) + (sensor == 0 ? 0.0 : phase[c]);
    return e.vib_amp[c] * sin(arg);
  }
  if (e.vib_type == 3)
    return e.series[(run_local * 3 + c) * e.series_len + (t % static_cast<uint32_t>(e.series_len))];
  return 0.0;
}

// phase A in Monte-Carlo mode for one sample: the six Box-Muller pairs are drawn in ONE
// straight-line block (six independent Philox -> log/sqrt/sincospi chains the scheduler can
// interleave), then (ref + b) + white [+ vib] per axis, and the GM drive normals.
template <class P>
__device__ __forceinline__ void noisy_sample(const P& p, const double* ref_a3,
                                             const double* ref_g3, uint32_t t, uint32_t run_lo,
                                             uint32_t run_hi, int64_t run_local,
                                             const double* phase, double* ma, double* mg,
                                             double* za, double* zg) {
  Normal2 z[6];
#pragma unroll
  for (int c = 0; c < 6; ++c) z[c] = normal_pair(t, c, run_lo, run_hi, p.k0, p.k1);  // draws 0..5
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    za[c] = z[c].z0;
    zg[c] = z[3 + c].z0;
    ma[c] = (ref_a3[c] + p.accel.b[c]) + p.accel.w[c] * z[c].z1;
    mg[c] = (ref_g3[c] + p.gyro.b[c]) + p.gyro.w[c] * z[3 + c].z1;
  }
  if (p.accel.vib_type | p.gyro.vib_type) {   // uniform branch, off in the BASELINE configs
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      ma[c] += vib_term(p.accel, c, 0, t, run_lo, run_hi, p.k0, p.k1, run_local, phase);
      mg[c] += vib_term(p.gyro, c, 1, t, run_lo, run_hi, p.k0, p.k1, run_local, phase);
    }
  }
}

// Gauss-Markov drift of the G samples of a block, time-parallel: d[t+1] = a d[t] + b z[t] is an
// affine recurrence, so the group runs an inclusive scan y_j = sum_{q<=j} a^(j-q) b z_q with
// warp shuffles; d_j = a^j carry + y_(j-1) and the carry moves on by a^G carry + y_(G-1).
template <int G>
__device__ __forceinline__ double gm_block(double x, double a, double apj, double aG, int j,
                                           double& carry) {
  double y = x;
  if (G > 1) {
    double ap = a;
#pragma unroll
    for (int off = 1; off < G; off <<= 1) {
      const double u = __shfl_up_sync(0xffffffffu, y, off, G);
      if (j >= off) y = fma(ap, u, y);
      ap *= ap;
    }
  }
  double ym1 = 0.0, ylast = y;
  if (G > 1) {
    ym1 = __shfl_up_sync(0xffffffffu, y, 1, G);
    if (j == 0) ym1 = 0.0;
    ylast = __shfl_sync(0xffffffffu, y, G - 1, G);
  }
  const double d = (G > 1) ? fma(apj, carry, ym1) : carry;
  carry = fma(aG, carry, ylast);
  return d;
}

// Row of sample t in the (possibly decimated) histories; false: the sample is not kept.
__device__ __forceinline__ bool dump_row_generic(int64_t stride, int64_t t, int64_t* row) {
  if (stride <= 1) {
    *row = t;
    return true;
  }
  const int64_t q = t / stride;
  *row = q;
  return q * stride == t;
}
__device__ __forceinline__ bool dump_row(const McParams& p, int64_t t, int64_t* row) {
  return dump_row_generic(p.dump_stride, t, row);
}

// attitude.euler2quat, 'zyx' (attitude.py:188-205): [yaw, pitch, roll] -> scalar-first quaternion
__device__ __forceinline__ void write_quat(double* q, double yaw, double pitch, double roll) {
  double sy, cy, sp, cp, sr, cr;
  sincos_angle(0.5 * yaw, &sy, &cy);
  sincos_angle(0.5 * pitch, &sp, &cp);
  sincos_angle(0.5 * roll, &sr, &cr);
  q[0] = cy * cp * cr + sy * sp * sr;
  q[1] = cy * cp * sr - sy * sp * cr;
  q[2] = cy * sp * cr + sy * cp * sr;
  q[3] = sy * cp * cr - cy * sp * sr;
}

// ---- the per-run skeleton of the three Monte-Carlo kernels ------------------------------------------
// The run a lane works on, from its place in the grid (run_raw).
struct McRun {
  int64_t run;       // the run of this launch; groups past the last run shadow it (and write nothing)
  uint32_t lo, hi;   // the global run id (Philox key words)
  bool active;       // run_raw is a run of this launch
  bool dump;         // the run's histories are written
  bool warp_dumps;   // some lane of the warp writes histories
};
__device__ __forceinline__ McRun mc_run(const McParams& p, int64_t run_raw) {
  McRun r;
  r.active = run_raw < p.runs;
  r.run = r.active ? run_raw : p.runs - 1;
  const int64_t grun = p.run_offset + r.run;
  r.lo = static_cast<uint32_t>(grun);
  r.hi = static_cast<uint32_t>(grun >> 32);
  r.dump = r.active && r.run < p.dump_runs;
  r.warp_dumps = __any_sync(0xffffffffu, r.dump);
  return r;
}

// sample 0 of a run: its initial-state set (free_integration.py:85-87: one set for every run, or one each)
template <int RF>
__device__ __forceinline__ NavState mc_init(const McParams& p, int64_t run) {
  NavState st;
  const int64_t irun = p.ini_offset + run;
  const int64_t set = (irun < p.ini_sets) ? irun : 0;
  nav_init<RF>(st, p.ini + set * p.ini_rows, p.ini_rows, p.dt);
  return st;
}

// History rows: the attitude (and its quaternion), position and velocity of one kept sample
__device__ __forceinline__ void put_att_row(const McParams& p, int64_t run, int64_t row, double yaw, double pitch,
                                            double roll) {
  const int64_t o = run * p.osr + row * p.ost;
  p.out_att[o] = yaw;
  p.out_att[o + p.osc] = pitch;
  p.out_att[o + 2 * p.osc] = roll;
  if (p.out_quat) write_quat(p.out_quat + (run * p.dump_rows + row) * 4, yaw, pitch, roll);
}
__device__ __forceinline__ void put_pv_row(const McParams& p, int64_t run, int64_t row, const Vec3& pos,
                                           const Vec3& vel) {
  const int64_t o = run * p.osr + row * p.ost;
  p.out_pos[o] = pos.x;
  p.out_pos[o + p.osc] = pos.y;
  p.out_pos[o + 2 * p.osc] = pos.z;
  p.out_vel[o] = vel.x;
  p.out_vel[o + p.osc] = vel.y;
  p.out_vel[o + 2 * p.osc] = vel.z;
}
__device__ __forceinline__ void put_state_row(const McParams& p, int64_t run, int64_t row, double yaw, double pitch,
                                              double roll, const Vec3& pos, const Vec3& vel) {
  put_pv_row(p, run, row, pos, vel);
  put_att_row(p, run, row, yaw, pitch, roll);
}

// Lane k of a group keeps the state after step k of a pass (the outputs' wrap applied) ...
__device__ __forceinline__ void keep_state(double* keep, const NavState& st) {
  keep[0] = wrap_once(st.yaw); keep[1] = st.pitch; keep[2] = wrap_once(st.roll);
  keep[3] = st.pos.x; keep[4] = st.pos.y; keep[5] = st.pos.z;
  keep[6] = st.vel.x; keep[7] = st.vel.y; keep[8] = st.vel.z;
}
// ... and writes it after the pass as the row of sample t + 1 (t: the lane's sample of the pass)
__device__ __forceinline__ void put_kept_row(const McParams& p, int64_t run, int64_t t, const double* keep) {
  int64_t row;
  if (p.out_att && t + 1 < p.n && dump_row(p, t + 1, &row))
    put_state_row(p, run, row, keep[0], keep[1], keep[2], Vec3{keep[3], keep[4], keep[5]},
                  Vec3{keep[6], keep[7], keep[8]});
}

// Per-run results at the last sample: the end-point error against the reference (angles by
// angle_range_pi) and the end state (yaw and roll wrapped once); ATT: the attitude part, PV: position, velocity
template <bool ATT, bool PV>
__device__ __forceinline__ void put_end(const McParams& p, int64_t run, double yaw, double pitch, double roll,
                                        const Vec3& pos, const Vec3& vel) {
  if (p.end_err) {
    const double* r = p.ref_nav + (p.n - 1) * 9;
    double* e = p.end_err + run * 9;
    if (ATT) {
      e[0] = angle_range_pi(yaw - r[0]);
      e[1] = angle_range_pi(pitch - r[1]);
      e[2] = angle_range_pi(roll - r[2]);
    }
    if (PV) {
      e[3] = pos.x - r[3];
      e[4] = pos.y - r[4];
      e[5] = pos.z - r[5];
      e[6] = vel.x - r[6];
      e[7] = vel.y - r[7];
      e[8] = vel.z - r[8];
    }
  }
  if (p.end_state) {
    double* e = p.end_state + run * 9;
    if (ATT) {
      e[0] = wrap_once(yaw); e[1] = pitch; e[2] = wrap_once(roll);
    }
    if (PV) {
      e[3] = pos.x; e[4] = pos.y; e[5] = pos.z;
      e[6] = vel.x; e[7] = vel.y; e[8] = vel.z;
    }
  }
}

// Process errors of one sample against the truth row r [9] (ins_data_manager.py:536-541), one column group
// at a time (K12 takes all three, K7 gives each to one lane of a run): the attitude through angle_range_pi,
// the velocity as plain differences.
__device__ __forceinline__ void proc_err_att(const NavState& st, const double* r, double* e) {
  e[0] = angle_range_pi(st.yaw - r[0]);
  e[1] = angle_range_pi(st.pitch - r[1]);
  e[2] = angle_range_pi(st.roll - r[2]);
}
// The position: LLA differences, or in ref_frame 0 with a non-zero pos_frame (uniform over the launch) in
// metres, as array_error does for extra_opt 'ned' / 'ecef' (:543-552): d = lla2ecef(x) - lla2ecef(r), and for
// NED c_ne(r) . d.  Both points are converted from their LLA values, not from the step's carried latitude
// sin/cos.
template <int RF>
__device__ __forceinline__ void proc_err_pos(const NavState& st, const double* r, int pos_frame, double* e) {
  if (RF == 0 && pos_frame != 0) {
    const Vec3 x = lla2ecef(st.pos.x, st.pos.y, st.pos.z);
    const Vec3 xr = lla2ecef(r[3], r[4], r[5]);
    const Vec3 d{x.x - xr.x, x.y - xr.y, x.z - xr.z};
    if (pos_frame == 1) {   // attitude.ecef_to_ned(lat, lon) of the truth
      double sl, cl, so, co;
      sincos_angle(r[3], &sl, &cl);
      sincos_angle(r[4], &so, &co);
      e[0] = -sl * co * d.x - sl * so * d.y + cl * d.z;
      e[1] = -so * d.x + co * d.y;
      e[2] = -cl * co * d.x - cl * so * d.y - sl * d.z;
    } else {
      e[0] = d.x;
      e[1] = d.y;
      e[2] = d.z;
    }
  } else {
    e[0] = st.pos.x - r[3];
    e[1] = st.pos.y - r[4];
    e[2] = st.pos.z - r[5];
  }
}
__device__ __forceinline__ void proc_err_vel(const NavState& st, const double* r, double* e) {
  e[0] = st.vel.x - r[6];
  e[1] = st.vel.y - r[7];
  e[2] = st.vel.z - r[8];
}

// Adds the NC errors e to the accumulators max|e|, shifted sum, shifted sum of squares and shift K (the first
// error sample, taken when `first`); column c of each accumulator is at [c * S].
//
// The shift keeps the one-pass variance sq / n - (sum / n)^2 from cancelling when the errors sit far from 0:
// its relative error grows with n and with the distance of the first sample from the others (with the first
// sample 1e6 standard deviations away, ~5e-9 at n = 2e5; tests/test_gpu_stats_edges.py holds it to 1e-8).
// The loop runs on every sample, so it is left as it is (fmax included): proc_put recovers NumPy's non-finite
// results from the sums and the shift (see there).  `first` is not a branch taken once: the compiler turns it
// into selects on every sample, and a finite-shift select there (K = isfinite(e) ? e : 0) made the K12 PROC
// launch ~2% slower (1000 runs x 1000 samples, H100 80GB HBM3 at 700 W: 1.150 against 1.124 ms).
template <int NC, int S>
__device__ __forceinline__ void proc_fold(const double* e, bool first, double* mx, double* sum, double* sq,
                                          double* k) {
  if (first) {
#pragma unroll
    for (int c = 0; c < NC; ++c) k[c * S] = e[c];
  }
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    mx[c * S] = fmax(mx[c * S], fabs(e[c]));
    const double d = e[c] - k[c * S];
    sum[c * S] += d;
    sq[c * S] += d * d;
  }
}

// max|e|, mean and std (ddof 0) of NC accumulated columns into o[c], o[9 + c], o[18 + c] (the [3][9] rows of
// proc_stats); inv = 1 / the sample count, NaN for no samples (all three statistics are then NaN).
// NumPy's non-finite rules, from the sums: with a finite shift K, a NaN sample makes sq NaN, and then max,
// mean and std are NaN; +-inf samples make sq = +inf, mean = +-inf (NaN for both signs), std =
// sqrt(inf - inf) = NaN, and max = inf from the fmax of the loop.  A NaN K (a NaN first sample) makes
// everything NaN.  A +-inf K (an infinite first sample) makes the sums NaN; max is then inf, mean K and std
// NaN, NumPy's results unless the column also holds a NaN or the other infinity (which one pass cannot see).
template <int NC, int S>
__device__ __forceinline__ void proc_put(double* o, double inv, const double* mx, const double* sum,
                                         const double* sq, const double* k) {
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const double kc = k[c * S];
    const bool kinf = isinf(kc);
    const double m = sum[c * S] * inv;  // mean of (e - K)
    const double q = sq[c * S] * inv;   // NaN iff a NaN sample, no samples or a +-inf K
    o[c] = (q != q && !kinf) ? q : mx[c * S];
    o[9 + c] = kinf ? kc : kc + m;
    const double v = q - m * m;
    o[18 + c] = sqrt(v < 0.0 ? 0.0 : v);
  }
}

// process-error accumulation of one sample (ins_data_manager.py:536-541, :761-808) over all nine columns
template <int RF>
__device__ __forceinline__ void proc_accumulate(const NavState& st, const double* r, int pos_frame,
                                                double* pe_max, double* pe_sum, double* pe_sq, double* pe_k,
                                                int64_t& pe_cnt) {
  double e[9];
  proc_err_att(st, r, e);
  proc_err_pos<RF>(st, r, pos_frame, e + 3);
  proc_err_vel(st, r, e + 6);
  proc_fold<9, 1>(e, pe_cnt == 0, pe_max, pe_sum, pe_sq, pe_k);
  ++pe_cnt;
}

// a^e for a small non-negative integer e (binary powering; no libm call, no stack frame)
__device__ __forceinline__ double ipow(double a, int e) {
  double r = 1.0, b = a;
#pragma unroll
  for (int bit = 0; bit < 6; ++bit) {
    if ((e >> bit) & 1) r *= b;
    b *= b;
  }
  return r;
}

// resident CTAs per SM the register allocation must allow: the throughput configuration
// (G = 1) wants many warps per scheduler to cover FP64 latency; wide groups are latency bound
// by the serial recurrence and keep their registers
#ifndef B2INS_G1_MINBLOCKS
#define B2INS_G1_MINBLOCKS 5   // tools/variants.sh times 3 / 4 / 5
#endif
template <int G>
struct MinBlocks {
  static constexpr int value = (G == 1) ? B2INS_G1_MINBLOCKS : (G == 2 ? 3 : 2);
};

// (The warp-specialised forms of the fused launch are mc_spec_kernel.cuh and mc_av_kernel.cuh.)
template <int G, int RF, bool FED, bool PROC>
__global__ void __launch_bounds__(kThreads, MinBlocks<G>::value)
mc_kernel(const __grid_constant__ McParams p) {
  __shared__ TileSmem<PROC> sm;
  constexpr int kRunsPerWarp = 32 / G;
  constexpr bool kSplit = (G >= 4);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int j = lane % G;
  const int role = lane & 3;
  const McRun mr = mc_run(p, (static_cast<int64_t>(blockIdx.x) * kWarps + warp) * kRunsPerWarp + lane / G);
  const bool odo_mode = p.algo == 1;
  constexpr bool kStaged = !FED || PROC;
  constexpr int kStages = Stages<PROC>::value;

  const int64_t num_tiles = (p.n + kTile - 1) / kTile;
  if (kStaged) {
    if (threadIdx.x == 0) {
      for (int s = 0; s < kStages; ++s) {
        mbar_init(&sm.full[s], 1);
        mbar_init(&sm.empty[s], kWarps);
      }
      mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int s = 0; s < kStages && s < num_tiles; ++s) issue_tile<FED, PROC>(sm, p, s, s);
    }
  }

  // ---- sample 0 ----------------------------------------------------------
  NavState st = mc_init<RF>(p, mr.run);
  // Gauss-Markov drift carried across blocks (d[0] = 0), and the powers a^j, a^G
  double carry[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  double apj[6], aG[6];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double aa = p.accel.gm_a[c], ag = p.gyro.gm_a[c];
    apj[c] = (G > 1) ? ipow(aa, j) : 1.0;
    apj[3 + c] = (G > 1) ? ipow(ag, j) : 1.0;
    aG[c] = (G > 1) ? ipow(aa, G) : aa;
    aG[3 + c] = (G > 1) ? ipow(ag, G) : ag;
  }
  double phase[3] = {0.0, 0.0, 0.0};
  if (!FED && p.gyro.vib_type == 2) {
#pragma unroll
    for (int c = 0; c < 3; ++c)  // np.random.rand(1)*2*pi, pathgen.py:553-555
      phase[c] = (uniform01(0xFFFFFFFFu, kDrawPhase + c, mr.lo, mr.hi, p.k0, p.k1) * 2.0) * kPi;
  }
  if (mr.dump && j == 0 && p.out_att) put_state_row(p, mr.run, 0, st.yaw, st.pitch, st.roll, st.pos, st.vel);
  // process-error accumulators (shifted sums: K = first error sample)
  double pe_max[9], pe_sum[9], pe_sq[9], pe_k[9];
  int64_t pe_cnt = 0;
  if (PROC) {
#pragma unroll
    for (int c = 0; c < 9; ++c) pe_max[c] = pe_sum[c] = pe_sq[c] = pe_k[c] = 0.0;
  }

  // ---- time loop ---------------------------------------------------------
  for (int64_t tile = 0; tile < num_tiles; ++tile) {
    const int s = static_cast<int>(tile % kStages);
    const uint32_t parity = static_cast<uint32_t>((tile / kStages) & 1);
    const int64_t t0 = tile * kTile;
    const int cnt = static_cast<int>(min64(kTile, p.n - t0));
    if (kStaged)
      refill_and_wait<FED, PROC>(sm, p, threadIdx.x == 0, static_cast<int>(tile),
                                 static_cast<int>(num_tiles), s, parity, 0);

    for (int base = 0; base < cnt; base += G) {
      B2_CLK(ca0);
      // ---------------- phase A: lane j prepares sample t0 + base + j --------------
      double mg[3], ma[3];  // the complete measurement of sample base + j
      double mo = 0.0;      // odometer measurement (algo 1)
      const int tj = base + j;
      const int64_t t = t0 + tj;
      {
      if (FED) {
        if (tj < cnt) {
          const int64_t o = mr.run * p.sr + t * p.st;
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            mg[c] = p.fed_gyro[o + c * p.sc];
            ma[c] = odo_mode ? 0.0 : p.fed_accel[o + c * p.sc];
          }
          if (odo_mode) mo = p.fed_odo[mr.run * p.so_r + t * p.so_t];
        } else {
#pragma unroll
          for (int c = 0; c < 3; ++c) mg[c] = ma[c] = 0.0;
        }
      } else {
        double zg[3], za[3];
        if (tj < cnt) {
          noisy_sample(p, &sm.accel[s][tj * 3], &sm.gyro[s][tj * 3], static_cast<uint32_t>(t), mr.lo,
                       mr.hi, mr.run, phase, ma, mg, za, zg);
        } else {
#pragma unroll
          for (int c = 0; c < 3; ++c) mg[c] = ma[c] = zg[c] = za[c] = 0.0;
        }
        B2_CLK(ca1);
        B2_ACC(1, ca0, ca1);
        // + drift: the GM state d[t] (pathgen.py:583-590) or drift*z[t] if tau = inf (:591-593)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const double da = gm_block<G>(p.accel.gm_b[c] * za[c], p.accel.gm_a[c], apj[c], aG[c], j,
                                        carry[c]);
          const double dg = gm_block<G>(p.gyro.gm_b[c] * zg[c], p.gyro.gm_a[c], apj[3 + c],
                                        aG[3 + c], j, carry[3 + c]);
          ma[c] += da + p.accel.wd[c] * za[c];
          mg[c] += dg + p.gyro.wd[c] * zg[c];
        }
        if (odo_mode) {   // pathgen.odo_gen, pathgen.py:627-641: scale*ref + stdv*randn
          const double zo = (tj < cnt) ? normal_pair(static_cast<uint32_t>(t), kDrawOdo, mr.lo, mr.hi,
                                                     p.k0, p.k1).z0 : 0.0;
          mo = (tj < cnt) ? p.odo_scale * p.ref_odo[t] + p.odo_stdv * zo : 0.0;
        }
      }
      int64_t row;
      if (mr.warp_dumps && mr.dump && tj < cnt && p.out_gyro && dump_row(p, t, &row)) {
        const int64_t o = mr.run * p.osr + row * p.ost;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          p.out_gyro[o + c * p.osc] = mg[c];
          p.out_accel[o + c * p.osc] = ma[c];
        }
        if (odo_mode && p.out_odo) p.out_odo[mr.run * p.dump_rows + row] = mo;
      }
      if (odo_mode) {   // the odometer sample rides to phase B in the accel.x slot
        ma[0] = mo;
        ma[1] = ma[2] = 0.0;
      }
      if (G > 1) {
        SampleSlot& mine = sm.slot[warp][lane];
        mine.g[0] = mg[0]; mine.g[1] = mg[1]; mine.g[2] = mg[2];
        mine.a[0] = ma[0]; mine.a[1] = ma[1]; mine.a[2] = ma[2];
      }
      }
      // hand-over from phase A to phase B: one warp doing both only needs its own lanes
      if (G > 1) __syncwarp();

      B2_CLK(cb0);
      B2_ACC(2, ca0, cb0);
      // ---------------- phase B: serial over the G samples of the block ------------
      double keep[9];  // lane k keeps the state after sample base+k (history output)
#pragma unroll
      for (int c = 0; c < 9; ++c) keep[c] = 0.0;
      // samples of this block that are followed by a step (the last sample of the series is not)
      const int kmax = static_cast<int>(min64(min64(G, cnt - base), p.n - 1 - (t0 + base)));
      const SampleSlot* grp = &sm.slot[warp][lane - j];
      // One step of the recurrence; HIST keeps the state after sample base+k in lane k.
      auto one_step = [&](int k, bool hist) {
        Vec3 w, f;
        if (G == 1) {
          w = Vec3{mg[0], mg[1], mg[2]};
          f = Vec3{ma[0], ma[1], ma[2]};
        } else {
          const SampleSlot& sl = grp[k];
          w = Vec3{sl.g[0], sl.g[1], sl.g[2]};
          f = Vec3{sl.a[0], sl.a[1], sl.a[2]};
        }
        if (PROC) {
          // error of sample t0+base+k (state BEFORE the step), ins_data_manager.py:536-541
          if (t0 + base + k >= p.stats_start)
            proc_accumulate<RF>(st, &sm.nav[s][(base + k) * 9], p.proc_pos_frame, pe_max, pe_sum, pe_sq,
                                pe_k, pe_cnt);
        }
        // exact trigonometry again after every kResync-th sample (a rule in absolute time: the same for
        // every lane-group width)
        const bool resync = ((t0 + base + k + 1) & (kResync - 1)) == 0;
        nav_step<RF, kSplit, 2>(st, w, f, p.dt, p.earth_rot != 0, role, resync, odo_mode);
        if (hist && j == k) keep_state(keep, st);
      };
      if (mr.warp_dumps) {         // history output: the rare path keeps the simple loop
#pragma unroll 1
        for (int k = 0; k < kmax; ++k) one_step(k, true);
      } else {
        // two steps per iteration: the off-chain tail of step k (velocity, position) overlaps the
        // dependency chain of step k+1 (ptxas does not pipeline across iterations by itself)
        int k = 0;
#pragma unroll 1
        for (; k + 1 < kmax; k += 2) {
          one_step(k, false);
          one_step(k + 1, false);
        }
        if (k < kmax) one_step(k, false);
      }
      if (G > 1) __syncwarp();   // slots are rewritten by the next block
      B2_CLK(cb1);
      B2_ACC(3, cb0, cb1);
      // ---------------- histories: lane j writes the state of sample base+j+1 ---------
      if (mr.warp_dumps && mr.dump && tj < cnt) put_kept_row(p, mr.run, t, keep);
    }

    if (kStaged) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.empty[s]);
    }
  }

  // ---- per-run results -----------------------------------------------------
  if (PROC) {   // the last sample has no step after it: its error is accumulated here
    if (p.n - 1 >= p.stats_start)
      proc_accumulate<RF>(st, p.ref_nav + (p.n - 1) * 9, p.proc_pos_frame, pe_max, pe_sum, pe_sq, pe_k,
                          pe_cnt);
  }
  if (mr.active && j == 0) {
    put_end<true, true>(p, mr.run, st.yaw, st.pitch, st.roll, st.pos, st.vel);
    if (PROC && p.proc_stats) {
      double* o = p.proc_stats + mr.run * 27;
      const double inv = pe_cnt > 0 ? 1.0 / static_cast<double>(pe_cnt) : __longlong_as_double(0x7ff8000000000000LL);
      proc_put<9, 1>(o, inv, pe_max, pe_sum, pe_sq, pe_k);
    }
  }
}

}  // namespace b2ins
