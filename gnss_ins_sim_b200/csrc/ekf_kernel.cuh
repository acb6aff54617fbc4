// K7: Monte-Carlo loosely-coupled GNSS/INS filter (BASELINE config 5).
//
// The reference's demo_algorithms/ins_loose.py is a stub (prediction() / correction() are `pass`,
// ins_loose.py:124-134): there is nothing to be parity-checked against.  The filter implemented here
// is specified from first principles in DESIGN.md section 11 (read that first: state order, error
// convention, Phi, Q, the six scalar GPS updates, the closed-loop correction); this kernel restates
// it for the device and is held to that spec on identical Philox draws.  What comes from the reference:
// the sensor models that feed it (pathgen.acc_gen / gyro_gen :441-594, gps_gen :596-625, the same
// Philox streams as K12 / K6) and the strapdown step (free_integration.py:133-172 = nav_step<0>).
//
// Four lanes own one Monte-Carlo run for the whole series (the filter is serial in time and its GPS
// epochs are common to all runs, so a warp never diverges on them): the nominal state and the bias
// estimates are replicated over the four lanes, everything else is shared out -- the six Box-Muller
// pairs of a sample, the columns / rows of the covariance sweeps, the rows of the rank-one updates.  The
// 15 x 15 covariance lives in shared memory as P[element][run of the CTA] (14.4 KB per 32-thread CTA of
// eight runs; every warp access is bank-conflict-free).  Per IMU sample: six Box-Muller pairs, one
// strapdown step, and P <- Phi P Phi^T + Q done as two in-place sweeps that use the block structure of
// Phi (about 1100 FMA instead of 6750).  Per GPS sample (every fs / fs_gps steps): three more pairs, six
// scalar updates, the correction.
#pragma once
#include "mc_kernel.cuh"
#include "gps_kernel.cuh"

namespace b2ins {

constexpr int kEkfThreads = 32;
constexpr int kEkfN = 15;
constexpr uint32_t kDrawIni = 27;   // + j, t = 0xFFFFFFFE: the initial-state errors (DESIGN.md section 11)
constexpr int kAlignN = 10;         // alignment: accelerometer samples averaged for roll and pitch (ins_loose.py:72)
constexpr int kAlignGps = 2;        // EkfParams::align of B2INS_ALIGN_GPS: yaw is the fix row's course over ground

struct EkfParams {
  int64_t n, runs, run_offset, m;
  double dt;
  int earth_rot;
  uint32_t k0, k1;
  TriadNoise gyro, accel;          // the generator (pre-digested as for K12)
  const double* ref_gyro;          // [n][3]
  const double* ref_accel;         // [n][3]
  const double* ref_nav;           // [n][9] att, pos (LLA), vel (NED)
  const double* ref_gps;           // [m][6]
  const int64_t* gps_idx;          // [m] IMU sample index of every GPS row (ascending)
  const double* gps_vis;           // [m] 1 = visible
  double stdp[3], stdv[3];         // GPS noise of the generator [m], [m/s] = the filter's R
  double p0[15];
  double ini[9];                   // true initial LLA, body velocity, Euler angles
  double ag[3], qg[3], aa[3], qa[3];   // bias model: a and b^2 per axis
  double arw2dt[3], vrw2dt[3];
  double qv_extra, qphi_extra;     // model-mismatch random walks: vel_rw^2 dt, att_rw^2 dt
  int64_t stats_start;
  double* end_err;                 // [runs][9]
  double* end_bias;                // [runs][6]
  double* consist;                 // [runs][19]: NEES sums (pos, vel, att), inside-3-sigma counts [15], epochs
  double* out_att;                 // histories of runs [0, dump_runs): [dump_runs][rows][3]
  double* out_pos;
  double* out_vel;
  double* out_wb;
  double* out_ab;
  int64_t dump_runs, dump_stride, dump_rows;
  // supplied measurements (ekf_kernel<false, true>), run-major: gyro, accel [runs][n][3], gps [runs][m][6]
  const double* fed_gyro;
  const double* fed_accel;
  const double* fed_gps;
  int ini_draw;                    // 1: the initial state is ini + the P0 draw of the run; 0: ini itself
  // process-error statistics (ekf_kernel<VIB, false, true>): samples >= proc_start, position columns as
  // B2INS_POS_FRAME_* proc_pos_frame
  double* proc_stats;              // [runs][3][9] max|e|, mean, std of att, pos, vel
  int64_t proc_start;
  int proc_pos_frame;
  // alignment (DESIGN.md section 11): B2INS_ALIGN_* (0: off, the initial state is ini + the P0 draw); the given
  // yaw; P0 of the level N / E misalignment and of the given yaw; the gyro's arw^2 per axis
  int align;
  double align_yaw, align_p0[3], arw2[3];
  // run-to-run turn-on bias (ekf_kernel<..., RB>; DESIGN.md section 11): the 1-sigma of every generator channel
  // (accel x y z, gyro x y z), drawn per run and folded into the channel's constant bias; the bias estimates minus
  // the true biases at sample n - 1, [runs][6] gyro then accel (NULL: not written)
  double rb[6];
  double* end_bias_err;
};

// The GPS row an aligned run starts at: the latest visible row at sample <= kAlignN - 1, else the first
// visible row after it; -1 without a visible row in the series.  GPS rows and visibility are common to all runs.
__device__ __forceinline__ int64_t ekf_fix_row(const EkfParams& p) {
  int64_t f = -1;
  for (int64_t j = 0; j < p.m; ++j) {
    if (p.gps_idx[j] >= p.n) break;
    const bool late = p.gps_idx[j] > kAlignN - 1;
    if (late && f >= 0) break;
    if (p.gps_vis[j] > 0.0) {
      f = j;
      if (late) break;
    }
  }
  return f;
}

// First sample of an aligned run's filter: max(kAlignN - 1, the fix row's sample); n without a fix row
__device__ __forceinline__ int64_t ekf_align_start(const EkfParams& p, int64_t fix) {
  return fix < 0 ? p.n : max(static_cast<int64_t>(kAlignN - 1), p.gps_idx[fix]);
}

// 3 x 3 symmetric-positive NEES  e^T A^-1 e  via the adjugate
__device__ __forceinline__ double nees3(const double* a /* row-major 3x3 */, const double* e) {
  const double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
  const double c11 = a[0] * a[8] - a[2] * a[6], c12 = a[1] * a[6] - a[0] * a[7];
  const double c22 = a[0] * a[4] - a[1] * a[3];
  const double det = a[0] * c00 + a[1] * c01 + a[2] * c02;
  const double q = e[0] * (c00 * e[0] + c01 * e[1] + c02 * e[2]) + e[1] * (c01 * e[0] + c11 * e[1] + c12 * e[2]) +
                   e[2] * (c02 * e[0] + c12 * e[1] + c22 * e[2]);
  return q / det;
}

// n -> b DCM (attitude.euler2dcm 'zyx' layout) -> [yaw, pitch, roll]
__device__ __forceinline__ void dcm2euler(const Dcm& c, double* yaw, double* pitch, double* roll) {
  *yaw = atan2(c.c01, c.c00);
  *pitch = -asin(fmin(1.0, fmax(-1.0, c.c02)));
  *roll = atan2(c.c12, c.c22);
}

// c (n -> b) times (I + s [phi x]), s = +-1
__device__ __forceinline__ Dcm dcm_times_small(const Dcm& c, const double* phi, double s) {
  const double x = s * phi[0], y = s * phi[1], z = s * phi[2];
  // (I + [phi x]) = [[1, -z, y], [z, 1, -x], [-y, x, 1]]
  Dcm r;
  r.c00 = c.c00 + c.c01 * z - c.c02 * y;
  r.c01 = -c.c00 * z + c.c01 + c.c02 * x;
  r.c02 = c.c00 * y - c.c01 * x + c.c02;
  r.c10 = c.c10 + c.c11 * z - c.c12 * y;
  r.c11 = -c.c10 * z + c.c11 + c.c12 * x;
  r.c12 = c.c10 * y - c.c11 * x + c.c12;
  r.c20 = c.c20 + c.c21 * z - c.c22 * y;
  r.c21 = -c.c20 * z + c.c21 + c.c22 * x;
  r.c22 = c.c20 * y - c.c21 * x + c.c22;
  return r;
}

__device__ __forceinline__ void set_attitude(NavState& st, double yaw, double pitch, double roll, double dt) {
  st.yaw = yaw;
  st.pitch = pitch;
  st.roll = roll;
  resync_exact<0>(st);
  st.icp = rcp_nr(st.sc.cp) * dt;
}

// FOUR lanes per run (a quad): the nominal state is replicated, everything else is shared out --
// the six Box-Muller pairs of a sample (lane q makes channel q, lanes 0 and 1 also channels 4 and 5; the
// Gauss-Markov state of a channel lives in its owner), the columns / rows of the two covariance sweeps,
// the rows of the rank-one updates.  P[element][run of the CTA] in shared memory.
constexpr int kEkfQ = 4;
constexpr int kEkfRuns = kEkfThreads / kEkfQ;     // 8 runs per CTA

// Row (= column) of P that lane q works on in its m-th turn (m = 0..3, a compile-time constant after
// unrolling): lanes 0..2 take row q of the position, velocity, attitude and accelerometer-bias blocks,
// lane 3 takes the three gyro-bias rows and sits out the fourth turn (it repeats its first row and
// stores nothing).  A turn therefore has ONE block type on lanes 0..2, which makes the process-noise
// terms of the second sweep compile-time, and any two lanes of a half-warp differ by an odd number of
// rows / columns, which keeps every 64-bit access of a warp on distinct banks.
__device__ __forceinline__ int ekf_own(int q, int m) {
  const int blk = (m == 3) ? 4 : m;
  return (q < 3) ? 3 * blk + q : ((m < 3) ? 9 + m : 9);
}

// VIB: the vibration models of p.accel / p.gyro (vib_term's, added last to each measurement) are compiled
// in; the launch picks ekf_kernel<false> when both vib_types are B2INS_VIB_NONE, so that instantiation is
// the filter without any vibration code.
// FED: the filter runs on supplied measurements (p.fed_gyro / fed_accel / fed_gps) instead of generating
// them: no Philox draws besides the optional initial-state draw, no Gauss-Markov carry, no vibration (it is
// in the data).  Lane q reads the channels it would generate, so the quad shuffles that build f and w are
// the same; sample i + 1 and the next GPS row are loaded a step / an epoch before they are used.  The
// consistency record needs the true biases and is compiled out; end_err is written when ref_nav is given.
// Alignment (p.align, a uniform run-time flag): the run initialises itself from its measurements instead of
// ini + the P0 draw.  Lanes q < 3 sum their accelerometer channel over samples 0..kAlignN-1 (a separate pass
// with its own Gauss-Markov carries; the quad shuffles replicate the mean) for roll and pitch at kAlignN - 1;
// yaw is given or the course of the fix row's GPS velocity (the draws that row's update would use).  The
// attitude alone then propagates (att_step: no Earth or transport rate) to the start sample s0, where
// position and velocity are the fix row as measured and P is the per-run diagonal P0; the filter runs from
// s0 with the first GPS row after it.  History rows before the state exists are NaN, the consistency record
// takes epochs after s0 and the process statistics start at max(proc_start, s0).
// PROC: per-run process-error statistics (proc_stats), taken where history row i is written -- after the GPS
// update of sample i -- against ref_nav row i for i >= proc_start.  The nominal state is replicated, so lane
// q < 3 of a run takes column group q (attitude, position, velocity) with no shuffle; its accumulators live
// in shared memory behind P, as [12][32 lanes], and lane 0 writes the run's [3][9] at the end.
// FA (FED only): alignment is compiled in and on; on supplied data it is a compile-time choice, because the
// run-time flag costs the fed form spills (ptxas -v).
// RB (generated measurements only): every run draws its turn-on bias, p.rb[c] times z0 of run-error pair c % 3 of
// sensor c / 3 (K1's draw, run_err_normals), once per channel in the prologue of the channel's owner lane, which
// folds it into the channel's constant bias.  The consistency record's true bias and p.end_bias_err take each
// channel's folded bias from its owner by quad shuffle, as they take its drift.
template <bool VIB, bool FED, bool PROC, bool FA = false, bool RB = false>
__global__ void __launch_bounds__(kEkfThreads) ekf_kernel(const __grid_constant__ EkfParams p) {
  static_assert(!(VIB && FED), "supplied measurements carry their vibration already");
  static_assert(!(FED && RB), "supplied measurements carry their turn-on bias already");
  static_assert(FED || !FA, "generated measurements select the alignment at run time (p.align)");
  const bool aligned = FED ? FA : (p.align != 0);
  static_assert(!(FED && PROC), "supplied-data histories are on the host: their statistics are taken there");
  constexpr int kAcc = PROC ? 12 * kEkfThreads : 0;    // 3 KB: max, sum, sum of squares, shift, 3 columns each
  __shared__ double Psm[kEkfN * kEkfN * kEkfRuns + kAcc];      // 14.4 KB (+ 3 KB)
  const int lane = threadIdx.x;
  // lane = q * 8 + rs: the eight runs of a quad index are neighbours, so a warp's 64-bit accesses to
  // P[element][run] fall on distinct banks whether the four q's differ in the column (sweep 1) or in
  // the row (sweep 2: rows are 15 * 8 doubles apart, half a bank cycle)
  const int q = lane >> 3, rs = lane & 7;
  const int64_t run_raw = static_cast<int64_t>(blockIdx.x) * kEkfRuns + rs;
  const bool active = run_raw < p.runs;
  const int64_t run = active ? run_raw : p.runs - 1;
  const int64_t grun = p.run_offset + run;
  const uint32_t run_lo = static_cast<uint32_t>(grun), run_hi = static_cast<uint32_t>(grun >> 32);
  const bool dump = active && q == 0 && run < p.dump_runs && p.out_att;
  const double dt = p.dt;
  auto P = [&](int i, int j) -> double& { return Psm[(i * kEkfN + j) * kEkfRuns + rs]; };
  auto quad = [&](double v, int owner) { return __shfl_sync(0xffffffffu, v, owner * kEkfRuns + rs); };
  // PROC: this lane's accumulators, column c of max|e| / shifted sum / shifted sum of squares / shift at
  // acc[(0 | 3 | 6 | 9 + c) * 32]
  double* const acc = Psm + kEkfN * kEkfN * kEkfRuns + lane;
  if constexpr (PROC) {
#pragma unroll
    for (int j = 0; j < 12; ++j) acc[j * kEkfThreads] = 0.0;
  }

  // GPS noise of the generator: horizontal sigmas in radians with the radii at the FIRST reference
  // sample, as pathgen.gps_gen does (pathgen.py:617-620)
  double sdp0 = p.stdp[0], sdp1 = p.stdp[1];
  if (!FED && p.m > 0) {
    const GeoParam gp = geo_param(p.ref_gps[0], p.ref_gps[2]);
    sdp0 = div_nr(sdp0, gp.rm);
    sdp1 = div_nr(div_nr(sdp1, gp.rn), gp.cl);
  }

  // ---- initial covariance and nominal state: truth + a draw from P0 (aligned: at s0, below) -------
  NavState st;
  if (!aligned) {
    for (int m = 0; m < 4; ++m) {
      const int r = ekf_own(q, m);
      if (q < 3 || m < 3)
        for (int c = 0; c < kEkfN; ++c) P(r, c) = (r == c) ? p.p0[r] : 0.0;
    }
    double e0[10];
#pragma unroll
    for (int j = 0; j < 5; ++j) {
      Normal2 z{0.0, 0.0};        // FED without ini_draw: a zero draw through the same code
      if (!FED || p.ini_draw) z = normal_pair(0xFFFFFFFEu, kDrawIni + j, run_lo, run_hi, p.k0, p.k1);
      e0[2 * j] = z.z0;
      e0[2 * j + 1] = z.z1;
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) e0[i] *= sqrt(p.p0[i]);
    double ini[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) ini[i] = p.ini[i];
    nav_init<0>(st, ini, 9, dt);          // the TRUE initial state: st.vel = C^T v_body
    const GeoParam gp = geo_param(ini[0], ini[2]);
    st.pos.x += e0[0] / (gp.rm + ini[2]);
    st.pos.y += e0[1] / ((gp.rn + ini[2]) * gp.cl);
    st.pos.z -= e0[2];
    st.vel.x += e0[3];
    st.vel.y += e0[4];
    st.vel.z += e0[5];
    // C_hat(n->b) = C(n->b) (I + [phi x])
    const Dcm c = dcm_times_small(dcm_from_sincos(st.sc), e0 + 6, 1.0);
    double y, pt, r;
    dcm2euler(c, &y, &pt, &r);
    set_attitude(st, y, pt, r, dt);
  }
  double bg[3] = {0.0, 0.0, 0.0}, ba[3] = {0.0, 0.0, 0.0};       // bias estimates (replicated)
  // the generator's channels of this lane: c0 = q (accel x y z, gyro x), c1 = q + 4 (gyro y z) for q < 2
  const int c0 = q, c1 = q + 4;
  const bool two = q < 2;
  auto model = [&](int c, double* b, double* w, double* wd, double* ga, double* gb) {
    const TriadNoise& e = (c < 3) ? p.accel : p.gyro;
    const int ax = c % 3;
    *b = e.b[ax]; *w = e.w[ax]; *wd = e.wd[ax]; *ga = e.gm_a[ax]; *gb = e.gm_b[ax];
  };
  double b0, w0, wd0, ga0, gb0, b1, w1, wd1, ga1, gb1;
  model(c0, &b0, &w0, &wd0, &ga0, &gb0);
  model(two ? c1 : c0, &b1, &w1, &wd1, &ga1, &gb1);
  if constexpr (RB) {
    // lanes 2 and 3 draw channel c0 twice and drop the second, like their second chain
    const int cc = two ? c1 : c0;
    b0 += p.rb[c0] * run_err_normals(c0 / 3, c0 % 3, run_lo, run_hi, p.k0, p.k1).z0;
    b1 += p.rb[cc] * run_err_normals(cc / 3, cc % 3, run_lo, run_hi, p.k0, p.k1).z0;
  }
  double carry0 = 0.0, carry1 = 0.0;                              // d[i] of the lane's channels
  // vibration (VIB only) of the lane's accelerometer channel (axis q, lanes 0..2) and gyro channel (c0 of
  // lane 3: x; c1 of lanes 0 and 1: y, z; lane 2 computes axis z and drops it): amplitude, the PSD model's
  // row of the series, the sinusoidal model's random gyro phase
  const int vax = q < 3 ? q : 0, vgx = q == 3 ? 0 : (q < 2 ? q + 1 : 2);
  double vamp_a = 0.0, vamp_g = 0.0, vphase = 0.0;
  const double* vser_a = nullptr;
  const double* vser_g = nullptr;
  if constexpr (VIB) {
    vamp_a = p.accel.vib_amp[vax];
    vamp_g = p.gyro.vib_amp[vgx];
    if (p.accel.vib_type == 3) vser_a = p.accel.series + (run * 3 + vax) * p.accel.series_len;
    if (p.gyro.vib_type == 3) vser_g = p.gyro.series + (run * 3 + vgx) * p.gyro.series_len;
    if (p.gyro.vib_type == 2)
      vphase = (uniform01(0xFFFFFFFFu, kDrawPhase + vgx, run_lo, run_hi, p.k0, p.k1) * 2.0) * kPi;
  }
  double nees[3] = {0.0, 0.0, 0.0};
  int inside[kEkfN];
#pragma unroll
  for (int i = 0; i < kEkfN; ++i) inside[i] = 0;
  int epochs = 0;
  int64_t jg = 0;                          // next GPS row
  int64_t next_gps = p.m > 0 ? p.gps_idx[0] : -1;
  // FED: the lane's two channels of its run (lanes 2 and 3 read c0 twice and drop the second) and the run's
  // GPS rows; nx0 / nx1 hold sample i + 1 during step i, ng the next GPS row
  const double* fch0 = nullptr;
  const double* fch1 = nullptr;
  const double* fgps = nullptr;
  double nx0 = 0.0, nx1 = 0.0, ng[6];
  if constexpr (FED) {
    const int cc = two ? c1 : c0;
    fch0 = (c0 < 3) ? p.fed_accel + run * p.n * 3 + c0 : p.fed_gyro + run * p.n * 3 + (c0 - 3);
    fch1 = (cc < 3) ? p.fed_accel + run * p.n * 3 + cc : p.fed_gyro + run * p.n * 3 + (cc - 3);
    fgps = p.fed_gps + run * p.m * 6;
    nx0 = fch0[0];
    nx1 = fch1[0];
#pragma unroll
    for (int k = 0; k < 6; ++k) ng[k] = p.m > 0 ? fgps[k] : 0.0;
  }
  // the measurements of sample i (the K12 generator, shared out over the quad): lane q's channels c0, c1 into
  // m0, m1, whose Gauss-Markov drifts cr0, cr1 carry; FED: sample i, loaded a step before, and sample i + 1
  auto measure = [&](int64_t i, double& cr0, double& cr1, double& m0, double& m1) {
    if constexpr (FED) {
      // sample i was loaded during step i - 1; sample i + 1 <= n - 1 is loaded now, a step before its use
      m0 = nx0;
      m1 = nx1;
      nx0 = fch0[(i + 1) * 3];
      nx1 = fch1[(i + 1) * 3];
    } else {
      const uint32_t t = static_cast<uint32_t>(i);
      const double* ref0 = (c0 < 3) ? p.ref_accel + i * 3 + c0 : p.ref_gyro + i * 3 + (c0 - 3);
      const Normal2 z0 = normal_pair(t, static_cast<uint32_t>(c0), run_lo, run_hi, p.k0, p.k1);
      m0 = ((ref0[0] + b0) + w0 * z0.z1) + (cr0 + wd0 * z0.z0);
      cr0 = fma(ga0, cr0, gb0 * z0.z0);
      // every lane runs a second chain (lanes 2 and 3 repeat their first draw and drop the result): no
      // divergent branch, and the two Box-Muller chains of a lane interleave
      const int cc = two ? c1 : c0;
      const double* ref1 = (cc < 3) ? p.ref_accel + i * 3 + cc : p.ref_gyro + i * 3 + (cc - 3);
      const Normal2 z1 = normal_pair(t, static_cast<uint32_t>(cc), run_lo, run_hi, p.k0, p.k1);
      m1 = ((ref1[0] + b1) + w1 * z1.z1) + (cr1 + wd1 * z1.z0);
      cr1 = two ? fma(ga1, cr1, gb1 * z1.z0) : 0.0;
      if constexpr (VIB) {
        // vib_term's models (1 random, 2 sinusoidal, 3 series), added last as in oracle_np.sensor_gen.
        // Random: lane q < 3 draws pair kDrawVib + q, whose z0 is its own accelerometer axis and whose z1
        // (gyro axis q) belongs to lane (q + 3) & 3 -- one quad shuffle from lane (q + 1) & 3; lane 3's
        // draw is dropped
        const int ta = p.accel.vib_type, tg = p.gyro.vib_type;
        double va = 0.0, vg = 0.0;
        if ((ta == 1) | (tg == 1)) {
          const Normal2 zv = normal_pair(t, kDrawVib + vax, run_lo, run_hi, p.k0, p.k1);
          const double zvg = quad(zv.z1, (q + 1) & 3);
          if (ta == 1) va = vamp_a * zv.z0;
          if (tg == 1) vg = vamp_g * zvg;
        }
        if (ta == 2) va = vamp_a * sin(p.accel.vib_w * static_cast<double>(t) + 0.0);
        if (tg == 2) vg = vamp_g * sin(p.gyro.vib_w * static_cast<double>(t) + vphase);
        if (ta == 3) va = vser_a[t % static_cast<uint32_t>(p.accel.series_len)];
        if (tg == 3) vg = vser_g[t % static_cast<uint32_t>(p.gyro.series_len)];
        m0 += (q < 3) ? va : vg;
        m1 += vg;
      }
    }
  };
  int64_t i0 = 0;                          // first sample of the filter
  if (aligned) {
    // ---- alignment: levelling at kAlignN - 1, the attitude alone to s0 = i0, the state and P0 at s0 ---
    const int64_t jf = ekf_fix_row(p);
    i0 = ekf_align_start(p, jf);
    const double qnan = __longlong_as_double(0x7ff8000000000000LL);
    // the fix row as measured (uniform branch): the GPS draws its update would use; FED: the supplied row
    double fx[6];
    if (jf < 0) {
#pragma unroll
      for (int k = 0; k < 6; ++k) fx[k] = qnan;
    } else if constexpr (FED) {
#pragma unroll
      for (int k = 0; k < 6; ++k) fx[k] = fgps[jf * 6 + k];
    } else {
      Normal2 zz{0.0, 0.0};
      if (q < 3) zz = normal_pair(static_cast<uint32_t>(jf), kPairGps + q, run_lo, run_hi, p.k0, p.k1);
      double zn[6];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        zn[2 * j] = quad(zz.z0, j);
        zn[2 * j + 1] = quad(zz.z1, j);
      }
      const double* rg = p.ref_gps + jf * 6;
      fx[0] = rg[0] + sdp0 * zn[0];
      fx[1] = rg[1] + sdp1 * zn[1];
      fx[2] = rg[2] + p.stdp[2] * zn[2];
#pragma unroll
      for (int k = 0; k < 3; ++k) fx[3 + k] = rg[3 + k] + p.stdv[k] * zn[3 + k];
    }
    // levelling: the mean of accelerometer samples 0..kAlignN-1 (ins_loose.py:76-91)
    double asum = 0.0;
    {
      double l0 = 0.0, l1 = 0.0;
      for (int64_t i = 0; i < kAlignN; ++i) {
        double a0, a1;
        if constexpr (FED)
          a0 = fch0[i * 3];
        else
          measure(i, l0, l1, a0, a1);
        asum += a0;
      }
    }
    const double ax = quad(asum, 0) / kAlignN, ay = quad(asum, 1) / kAlignN, az = quad(asum, 2) / kAlignN;
    const double nrm = sqrt(ax * ax + ay * ay + az * az);
    AttState a;
    a.yaw = (p.align == kAlignGps) ? atan2(fx[4], fx[3]) : p.align_yaw;
    a.pitch = asin(ax / nrm);
    a.roll = atan2(-(ay / nrm), -(az / nrm));
    att_exact(a);
    a.icp = rcp_nr(a.sc.cp) * dt;
    for (int64_t i = 0; i < i0; ++i) {
      int64_t row;
      if (dump && dump_row_generic(p.dump_stride, i, &row)) {
        const int64_t o = (run * p.dump_rows + row) * 3;
        const bool up = i >= kAlignN - 1;
        p.out_att[o] = up ? wrap_once(a.yaw) : qnan;
        p.out_att[o + 1] = up ? a.pitch : qnan;
        p.out_att[o + 2] = up ? wrap_once(a.roll) : qnan;
#pragma unroll
        for (int c3 = 0; c3 < 3; ++c3) {
          p.out_pos[o + c3] = qnan;
          p.out_vel[o + c3] = qnan;
          p.out_wb[o + c3] = 0.0;
          p.out_ab[o + c3] = 0.0;
        }
      }
      if (i == p.n - 1) break;
      double m0, m1;
      measure(i, carry0, carry1, m0, m1);
      const Vec3 w{quad(m0, 3), quad(m1, 0), quad(m1, 1)};
      if (i >= kAlignN - 1) att_step(a, w, dt, ((i + 1) & (kResync - 1)) == 0);
    }
    // the state at s0: position and velocity as measured, the attitude with exact sin/cos (and the latitude's)
    st.pos = Vec3{fx[0], fx[1], fx[2]};
    st.vel = Vec3{fx[3], fx[4], fx[5]};
    st.vel_b = Vec3{0.0, 0.0, 0.0};
    st.g = 0.0;
    st.fixed_g = false;
    set_attitude(st, a.yaw, a.pitch, a.roll, dt);
    // P0 at s0 (diagonal): the level / yaw variances plus the gyro's growth over the gap, the rest as p0
    const double gap = static_cast<double>(i0 - (kAlignN - 1)) * dt;
    double yv = p.align_p0[2];
    if (p.align == kAlignGps) {
      const double vn = fx[3], ve = fx[4], h2 = vn * vn + ve * ve;
      yv = (p.stdv[0] * p.stdv[0] * (ve * ve) + p.stdv[1] * p.stdv[1] * (vn * vn)) / (h2 * h2);
    }
    for (int m = 0; m < 4; ++m) {
      const int r = ekf_own(q, m);
      double d = p.p0[r];
      if (r >= 6 && r < 9) {
        const int c = r - 6;
        d = ((c == 2) ? yv : p.align_p0[c]) + (p.arw2[c] * gap + p.p0[9 + c] * (gap * gap));
      }
      if (q < 3 || m < 3)
        for (int c = 0; c < kEkfN; ++c) P(r, c) = (r == c) ? d : 0.0;
    }
    if constexpr (PROC) {
      // statistics from proc_start < s0 start at s0: its error is the shift of the accumulators
      if (q < 3 && p.proc_start < i0 && i0 < p.n) {
        const double* rn9 = p.ref_nav + i0 * 9;
        double e[3];
        if (q == 0)
          proc_err_att(st, rn9, e);
        else if (q == 1)
          proc_err_pos<0>(st, rn9, p.proc_pos_frame, e);
        else
          proc_err_vel(st, rn9, e);
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[(9 + c) * kEkfThreads] = e[c];
      }
    }
    while (jg < p.m && p.gps_idx[jg] <= i0) ++jg;       // the fix row and those before it are used
    next_gps = jg < p.m ? p.gps_idx[jg] : -1;
    if constexpr (FED) {
#pragma unroll
      for (int k = 0; k < 6; ++k) ng[k] = jg < p.m ? fgps[jg * 6 + k] : 0.0;
    }
  }
  __syncwarp();

  for (int64_t i = i0; i < p.n; ++i) {
    // ================= GPS sample of IMU sample i: update, then the consistency record ==========
    if (i == next_gps) {
      if (p.gps_vis[jg] > 0.0) {
        double zn[6];
        if constexpr (!FED) {
          // the three GPS pairs: lane q < 3 makes pair q, the quad shares them
          Normal2 zz{0.0, 0.0};
          if (q < 3) zz = normal_pair(static_cast<uint32_t>(jg), kPairGps + q, run_lo, run_hi, p.k0, p.k1);
#pragma unroll
          for (int j = 0; j < 3; ++j) {
            zn[2 * j] = quad(zz.z0, j);
            zn[2 * j + 1] = quad(zz.z1, j);
          }
        }
        const double* rg = p.ref_gps + jg * 6;
        const GeoParam gp = geo_param_sc(st.sl, st.cl, st.pos.z);
        const double rmh = gp.rm + st.pos.z, rnh = (gp.rn + st.pos.z) * gp.cl;
        double zm[6];
        if constexpr (FED) {
          zm[0] = (st.pos.x - ng[0]) * rmh;
          zm[1] = (st.pos.y - ng[1]) * rnh;
          zm[2] = -(st.pos.z - ng[2]);
          zm[3] = st.vel.x - ng[3];
          zm[4] = st.vel.y - ng[4];
          zm[5] = st.vel.z - ng[5];
        } else {
          zm[0] = (st.pos.x - (rg[0] + sdp0 * zn[0])) * rmh;
          zm[1] = (st.pos.y - (rg[1] + sdp1 * zn[1])) * rnh;
          zm[2] = -(st.pos.z - (rg[2] + p.stdp[2] * zn[2]));
          zm[3] = st.vel.x - (rg[3] + p.stdv[0] * zn[3]);
          zm[4] = st.vel.y - (rg[4] + p.stdv[1] * zn[4]);
          zm[5] = st.vel.z - (rg[5] + p.stdv[2] * zn[5]);
        }
        double x[kEkfN];
#pragma unroll
        for (int c = 0; c < kEkfN; ++c) x[c] = 0.0;
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          // row k of P (= column k: P is symmetric), read by every lane before its owner rewrites it
          double row[kEkfN];
#pragma unroll
          for (int c = 0; c < kEkfN; ++c) row[c] = P(k, c);
          __syncwarp();
          const double rk = (k < 3) ? p.stdp[k] * p.stdp[k] : p.stdv[k - 3] * p.stdv[k - 3];
          const double inv_s = 1.0 / (row[k] + rk);
          const double innov = zm[k] - x[k];
#pragma unroll
          for (int c = 0; c < kEkfN; ++c) x[c] = fma(row[c] * inv_s, innov, x[c]);      // x += K innov, K = P[:,k] / s
          // P <- P - P[:,k] P[k,:] / s on this lane's rows.  The product P[a,k] P[b,k] is formed first, so
          // the (a,b) and (b,a) entries -- computed by different lanes -- get the same bits: the symmetric
          // result the spec reaches by (P + P^T) / 2
#pragma unroll
          for (int m = 0; m < 4; ++m) {
            const int a = ekf_own(q, m);
            const double pak = P(a, k);
            double v[kEkfN];
#pragma unroll
            for (int b = 0; b < kEkfN; ++b) v[b] = fma(-(pak * row[b]), inv_s, P(a, b));
            if (q < 3 || m < 3) {
#pragma unroll
              for (int b = 0; b < kEkfN; ++b) P(a, b) = v[b];
            }
          }
          __syncwarp();
        }
        // ---- close the loop (replicated) ------------------------------------------------------
        st.pos.x -= x[0] / rmh;
        st.pos.y -= x[1] / rnh;
        st.pos.z += x[2];
        st.vel.x -= x[3];
        st.vel.y -= x[4];
        st.vel.z -= x[5];
        // C(n->b) = C_hat(n->b) (I - [phi x])
        const Dcm c = dcm_times_small(dcm_from_sincos(st.sc), x + 6, -1.0);
        double y, pt, r;
        dcm2euler(c, &y, &pt, &r);
        set_attitude(st, y, pt, r, dt);     // also refreshes sin/cos of the corrected latitude
#pragma unroll
        for (int c3 = 0; c3 < 3; ++c3) {
          bg[c3] -= x[9 + c3];
          ba[c3] -= x[12 + c3];
        }
      }
      if (!FED && i >= p.stats_start) {
        // the generator's drift d[i] of every channel, from its owner
        double dch[6];
        dch[0] = quad(carry0, 0); dch[1] = quad(carry0, 1); dch[2] = quad(carry0, 2); dch[3] = quad(carry0, 3);
        dch[4] = quad(carry1, 0); dch[5] = quad(carry1, 1);
        // the generator's constant bias of every channel; RB: with the run's turn-on bias, from its owner
        double bch[6];
#pragma unroll
        for (int c3 = 0; c3 < 3; ++c3) {
          bch[c3] = p.accel.b[c3];
          bch[3 + c3] = p.gyro.b[c3];
        }
        if constexpr (RB) {
          bch[0] = quad(b0, 0); bch[1] = quad(b0, 1); bch[2] = quad(b0, 2); bch[3] = quad(b0, 3);
          bch[4] = quad(b1, 0); bch[5] = quad(b1, 1);
        }
        const double* rn9 = p.ref_nav + i * 9;
        const GeoParam gp = geo_param(rn9[3], rn9[5]);
        double e[kEkfN];
        e[0] = (st.pos.x - rn9[3]) * (gp.rm + rn9[5]);
        e[1] = (st.pos.y - rn9[4]) * (gp.rn + rn9[5]) * gp.cl;
        e[2] = -(st.pos.z - rn9[5]);
        e[3] = st.vel.x - rn9[6];
        e[4] = st.vel.y - rn9[7];
        e[5] = st.vel.z - rn9[8];
        const Dcm ct = dcm_from_sincos(sincos3(rn9[0], rn9[1], rn9[2]));    // true n -> b
        const Dcm ce = dcm_from_sincos(st.sc);                              // estimated n -> b
        // M = C_hat(b->n) C(n->b) = ce^T ct = I - [phi x]
        const double m21 = ce.c02 * ct.c01 + ce.c12 * ct.c11 + ce.c22 * ct.c21;
        const double m12 = ce.c01 * ct.c02 + ce.c11 * ct.c12 + ce.c21 * ct.c22;
        const double m02 = ce.c00 * ct.c02 + ce.c10 * ct.c12 + ce.c20 * ct.c22;
        const double m20 = ce.c02 * ct.c00 + ce.c12 * ct.c10 + ce.c22 * ct.c20;
        const double m10 = ce.c01 * ct.c00 + ce.c11 * ct.c10 + ce.c21 * ct.c20;
        const double m01 = ce.c00 * ct.c01 + ce.c10 * ct.c11 + ce.c20 * ct.c21;
        e[6] = -0.5 * (m21 - m12);
        e[7] = -0.5 * (m02 - m20);
        e[8] = -0.5 * (m10 - m01);
#pragma unroll
        for (int c3 = 0; c3 < 3; ++c3) {
          e[9 + c3] = bg[c3] - (bch[3 + c3] + dch[3 + c3]);
          e[12 + c3] = ba[c3] - (bch[c3] + dch[c3]);
        }
#pragma unroll
        for (int b = 0; b < 3; ++b) {
          double a9[9];
#pragma unroll
          for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c3 = 0; c3 < 3; ++c3) a9[r * 3 + c3] = P(3 * b + r, 3 * b + c3);
          nees[b] += nees3(a9, e + 3 * b);
        }
#pragma unroll
        for (int c = 0; c < kEkfN; ++c) inside[c] += (e[c] * e[c] <= 9.0 * P(c, c)) ? 1 : 0;      // |e| <= 3 sigma
        ++epochs;
      }
      ++jg;
      next_gps = jg < p.m ? p.gps_idx[jg] : -1;
      if constexpr (FED) {
        if (jg < p.m) {
#pragma unroll
          for (int k = 0; k < 6; ++k) ng[k] = fgps[jg * 6 + k];
        }
      }
    }
    // ================= histories ==================================================================
    int64_t row;
    if (dump && dump_row_generic(p.dump_stride, i, &row)) {
      const int64_t o = (run * p.dump_rows + row) * 3;
      p.out_att[o] = wrap_once(st.yaw); p.out_att[o + 1] = st.pitch; p.out_att[o + 2] = wrap_once(st.roll);
      p.out_pos[o] = st.pos.x; p.out_pos[o + 1] = st.pos.y; p.out_pos[o + 2] = st.pos.z;
      p.out_vel[o] = st.vel.x; p.out_vel[o + 1] = st.vel.y; p.out_vel[o + 2] = st.vel.z;
#pragma unroll
      for (int c3 = 0; c3 < 3; ++c3) {
        p.out_wb[o + c3] = bg[c3];
        p.out_ab[o + c3] = ba[c3];
      }
    }
    if constexpr (PROC) {
      // the state of history row i against truth row i (shared by all runs: it stays in L2)
      if (q < 3 && i >= p.proc_start) {
        const double* rn9 = p.ref_nav + i * 9;
        double e[3];
        if (q == 0)
          proc_err_att(st, rn9, e);
        else if (q == 1)
          proc_err_pos<0>(st, rn9, p.proc_pos_frame, e);
        else
          proc_err_vel(st, rn9, e);
        proc_fold<3, kEkfThreads>(e, i == p.proc_start, acc, acc + 3 * kEkfThreads, acc + 6 * kEkfThreads,
                                  acc + 9 * kEkfThreads);
      }
    }
    if (i == p.n - 1) break;
    // ================= the measurements of sample i (the K12 generator, shared out over the quad) ==
    double m0, m1;
    measure(i, carry0, carry1, m0, m1);
    const Vec3 f{quad(m0, 0) - ba[0], quad(m0, 1) - ba[1], quad(m0, 2) - ba[2]};
    const Vec3 w{quad(m0, 3) - bg[0], quad(m1, 0) - bg[1], quad(m1, 1) - bg[2]};
    // ================= covariance: P <- Phi P Phi^T + Q with the blocks of Phi ====================
    {
      const Dcm c = dcm_from_sincos(st.sc);          // n -> b of sample i; b -> n is its transpose
      const double cb[9] = {c.c00 * dt, c.c10 * dt, c.c20 * dt, c.c01 * dt, c.c11 * dt, c.c21 * dt,
                            c.c02 * dt, c.c12 * dt, c.c22 * dt};      // C(b->n) dt, row-major
      const Vec3 fn = rot_b2n(st.sc, f);
      const double sx = fn.x * dt, sy = fn.y * dt, sz = fn.z * dt;    // [f_n x] dt = [[0,-sz,sy],[sz,0,-sx],[-sy,sx,0]]
      // sweep 1, this lane's columns: A = Phi P
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const int j = ekf_own(q, m);
        double col[kEkfN];
#pragma unroll
        for (int r = 0; r < kEkfN; ++r) col[r] = P(r, j);
        double o[kEkfN];
        o[0] = fma(dt, col[3], col[0]);
        o[1] = fma(dt, col[4], col[1]);
        o[2] = fma(dt, col[5], col[2]);
        o[3] = col[3] + (-sz * col[7] + sy * col[8]) - (cb[0] * col[12] + cb[1] * col[13] + cb[2] * col[14]);
        o[4] = col[4] + (sz * col[6] - sx * col[8]) - (cb[3] * col[12] + cb[4] * col[13] + cb[5] * col[14]);
        o[5] = col[5] + (-sy * col[6] + sx * col[7]) - (cb[6] * col[12] + cb[7] * col[13] + cb[8] * col[14]);
        o[6] = col[6] + (cb[0] * col[9] + cb[1] * col[10] + cb[2] * col[11]);
        o[7] = col[7] + (cb[3] * col[9] + cb[4] * col[10] + cb[5] * col[11]);
        o[8] = col[8] + (cb[6] * col[9] + cb[7] * col[10] + cb[8] * col[11]);
#pragma unroll
        for (int c3 = 0; c3 < 3; ++c3) {
          o[9 + c3] = p.ag[c3] * col[9 + c3];
          o[12 + c3] = p.aa[c3] * col[12 + c3];
        }
        if (q < 3 || m < 3) {
#pragma unroll
          for (int r = 0; r < kEkfN; ++r) P(r, j) = o[r];
        }
      }
      __syncwarp();
      // Q of this lane's velocity and attitude rows (lanes 0..2): row q of C diag(vrw^2 dt) C^T and of
      // C diag(arw^2 dt) C^T (C = b -> n, here cb / dt), the model-mismatch random walks on the diagonal
      const double inv_dt2 = 1.0 / (dt * dt);
      double qv[3], qp[3];
      {
        double mycb[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) mycb[k] = (q == 0) ? cb[k] : ((q == 1) ? cb[3 + k] : cb[6 + k]);
        const double kv0 = mycb[0] * p.vrw2dt[0] * inv_dt2, kv1 = mycb[1] * p.vrw2dt[1] * inv_dt2,
                     kv2 = mycb[2] * p.vrw2dt[2] * inv_dt2;
        const double kp0 = mycb[0] * p.arw2dt[0] * inv_dt2, kp1 = mycb[1] * p.arw2dt[1] * inv_dt2,
                     kp2 = mycb[2] * p.arw2dt[2] * inv_dt2;
#pragma unroll
        for (int c3 = 0; c3 < 3; ++c3) {
          qv[c3] = kv0 * cb[c3 * 3] + kv1 * cb[c3 * 3 + 1] + kv2 * cb[c3 * 3 + 2];
          qp[c3] = kp0 * cb[c3 * 3] + kp1 * cb[c3 * 3 + 1] + kp2 * cb[c3 * 3 + 2];
        }
      }
      // sweep 2, this lane's rows: P = A Phi^T, + Q
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const int r = ekf_own(q, m);
        double a[kEkfN];
#pragma unroll
        for (int c2 = 0; c2 < kEkfN; ++c2) a[c2] = P(r, c2);
        double o[kEkfN];
        o[0] = fma(dt, a[3], a[0]);
        o[1] = fma(dt, a[4], a[1]);
        o[2] = fma(dt, a[5], a[2]);
        o[3] = a[3] + (-sz * a[7] + sy * a[8]) - (cb[0] * a[12] + cb[1] * a[13] + cb[2] * a[14]);
        o[4] = a[4] + (sz * a[6] - sx * a[8]) - (cb[3] * a[12] + cb[4] * a[13] + cb[5] * a[14]);
        o[5] = a[5] + (-sy * a[6] + sx * a[7]) - (cb[6] * a[12] + cb[7] * a[13] + cb[8] * a[14]);
        o[6] = a[6] + (cb[0] * a[9] + cb[1] * a[10] + cb[2] * a[11]);
        o[7] = a[7] + (cb[3] * a[9] + cb[4] * a[10] + cb[5] * a[11]);
        o[8] = a[8] + (cb[6] * a[9] + cb[7] * a[10] + cb[8] * a[11]);
#pragma unroll
        for (int c3 = 0; c3 < 3; ++c3) {
          o[9 + c3] = p.ag[c3] * a[9 + c3];
          o[12 + c3] = p.aa[c3] * a[12 + c3];
        }
        // the row's share of Q: m names the block of lanes 0..2, lane 3 holds gyro-bias row m
        if (m < 3) o[9 + m] += (q == 3) ? p.qg[m] : 0.0;
#pragma unroll
        for (int c3 = 0; c3 < 3; ++c3) {
          if (m == 1) o[3 + c3] = (q < 3) ? (o[3 + c3] + qv[c3]) + ((c3 == q) ? p.qv_extra : 0.0) : o[3 + c3];
          if (m == 2) o[6 + c3] = (q < 3) ? (o[6 + c3] + qp[c3]) + ((c3 == q) ? p.qphi_extra : 0.0) : o[6 + c3];
          if (m == 3) o[12 + c3] += (c3 == q) ? p.qa[c3] : 0.0;
        }
        if (q < 3 || m < 3) {
#pragma unroll
          for (int c2 = 0; c2 < kEkfN; ++c2) P(r, c2) = o[c2];
        }
      }
      __syncwarp();
    }
    // ================= nominal state (replicated) ===============================================
    const bool resync = ((i + 1) & (kResync - 1)) == 0;
    nav_step<0, false, 0>(st, w, f, dt, p.earth_rot != 0, 0, resync);
#pragma unroll
    for (int c3 = 0; c3 < 3; ++c3) {
      bg[c3] *= p.ag[c3];
      ba[c3] *= p.aa[c3];
    }
  }

  if constexpr (PROC) __syncwarp();       // lane 0 reads the accumulators of lanes 8 and 16 of its run
  // RB: the true bias of every channel at sample n - 1, b + b_run + d[n-1], from its owner
  double btrue[6];
  if constexpr (RB) {
    const double t0 = b0 + carry0, t1 = b1 + carry1;
    btrue[0] = quad(t0, 0); btrue[1] = quad(t0, 1); btrue[2] = quad(t0, 2); btrue[3] = quad(t0, 3);
    btrue[4] = quad(t1, 0); btrue[5] = quad(t1, 1);
  }
  if (active && q == 0) {
    if constexpr (PROC) {
      double* o = p.proc_stats + run * 27;
      const int64_t ps = p.align ? max(p.proc_start, ekf_align_start(p, ekf_fix_row(p))) : p.proc_start;
      // no fix in the series (ps = n): NaN statistics
      const double inv = ps < p.n ? 1.0 / static_cast<double>(p.n - ps) : __longlong_as_double(0x7ff8000000000000LL);
#pragma unroll
      for (int g = 0; g < 3; ++g) {
        const double* a = acc + g * kEkfRuns;          // lane g * 8 + rs
        proc_put<3, kEkfThreads>(o + 3 * g, inv, a, a + 3 * kEkfThreads, a + 6 * kEkfThreads, a + 9 * kEkfThreads);
      }
    }
    if (!FED || p.end_err) {
      const double* r = p.ref_nav + (p.n - 1) * 9;
      double* e = p.end_err + run * 9;
      e[0] = angle_range_pi(st.yaw - r[0]);
      e[1] = angle_range_pi(st.pitch - r[1]);
      e[2] = angle_range_pi(st.roll - r[2]);
      e[3] = st.pos.x - r[3];
      e[4] = st.pos.y - r[4];
      e[5] = st.pos.z - r[5];
      e[6] = st.vel.x - r[6];
      e[7] = st.vel.y - r[7];
      e[8] = st.vel.z - r[8];
    }
    if (p.end_bias) {
#pragma unroll
      for (int c3 = 0; c3 < 3; ++c3) {
        p.end_bias[run * 6 + c3] = bg[c3];
        p.end_bias[run * 6 + 3 + c3] = ba[c3];
      }
    }
    if (RB && p.end_bias_err) {
#pragma unroll
      for (int c3 = 0; c3 < 3; ++c3) {
        p.end_bias_err[run * 6 + c3] = bg[c3] - btrue[3 + c3];
        p.end_bias_err[run * 6 + 3 + c3] = ba[c3] - btrue[c3];
      }
    }
    if (!FED && p.consist) {
      double* o = p.consist + run * 19;
      o[0] = nees[0]; o[1] = nees[1]; o[2] = nees[2];
#pragma unroll
      for (int c = 0; c < kEkfN; ++c) o[3 + c] = static_cast<double>(inside[c]);
      o[18] = static_cast<double>(epochs);
    }
  }
}

}  // namespace b2ins
