// Strapdown free-integration mechanization: the per-timestep recurrence of
// FreeIntegration.run (demo_algorithms/free_integration.py:63-174) with the L1 math it
// calls (attitude.py:344-371 euler2dcm zyx, :679-721 euler_update_zyx, :758-770 cross3;
// geoparams.py:25-53 geo_param, :70-87 lla2ecef), written once for all kernels.
// The whole state lives in registers; everything is double.
#pragma once
#include "common.cuh"

// B2INS_HOST_TEST (tools/step_host.cu): the mechanization also compiles for the host, so that the
// step the kernels run, and their speculative block, are checked against the oracle on the CPU
// (tests/test_cpu_step.py, tests/test_cpu_exact_path.py)
#ifdef B2INS_HOST_TEST
#define B2_DEV __host__ __device__ __forceinline__
#else
#define B2_DEV __device__ __forceinline__
#endif

namespace b2ins {

struct Vec3 {
  double x, y, z;
};

// n -> b direction cosine matrix, row-major
struct Dcm {
  double c00, c01, c02, c10, c11, c12, c20, c21, c22;
};

struct SinCos3 {
  double sy, cy, sp, cp, sr, cr;  // yaw, pitch, roll
};

// sin/cos of an angle that normally lives in [-pi, pi] (Euler angles after their wrap,
// latitude, longitude).  sincos_bounded's three-term reduction stays accurate far beyond that:
// for 64 < |x| <= 1e6 the error is at most 2.5 ulp of the result + |q| 8.5e-32 absolute (q the
// quadrant index, up to 636 620; the second term is the split of pi/2 ending at PIO2_3, 5.4e-26 at
// 1e6), measured worst 2.39 ulp (tests/test_cpu_fastmath.py and, on the device, test_gpu_fastmath.py).
// Larger magnitudes are only reachable after the Euler-angle
// singularity at pitch = +-pi/2 has blown a rate up, where the recurrence is meaningless
// anyway -- they are mapped to the angle 0 by a select (branch-free, off the critical path).
// A NaN or an infinite angle maps to x - x = NaN, so its sin/cos are NaN as the reference's np.sin/np.cos
// are, and the run's later samples are NaN like the reference's (no fast-math: x - x is not folded to 0).
B2_DEV void sincos_angle(double x, double* s, double* c) {
  sincos_bounded(fabs(x) <= 1.0e6 ? x : x - x, s, c);
}

B2_DEV SinCos3 sincos3(double yaw, double pitch, double roll) {
  SinCos3 t;
  sincos_angle(yaw, &t.sy, &t.cy);
  sincos_angle(pitch, &t.sp, &t.cp);
  sincos_angle(roll, &t.sr, &t.cr);
  return t;
}

// attitude.euler2dcm, 'zyx' branch: attitude.py:361-371
B2_DEV Dcm dcm_from_sincos(const SinCos3& t) {
  Dcm c;
  c.c00 = t.cp * t.cy;
  c.c01 = t.cp * t.sy;
  c.c02 = -t.sp;
  c.c10 = t.sr * t.sp * t.cy - t.cr * t.sy;
  c.c11 = t.sr * t.sp * t.sy + t.cr * t.cy;
  c.c12 = t.cp * t.sr;
  c.c20 = t.sp * t.cr * t.cy + t.sy * t.sr;
  c.c21 = t.sp * t.cr * t.sy - t.cy * t.sr;
  c.c22 = t.cp * t.cr;
  return c;
}

B2_DEV Vec3 mul_t(const Dcm& c, const Vec3& v) {  // c^T . v
  return Vec3{c.c00 * v.x + c.c10 * v.y + c.c20 * v.z, c.c01 * v.x + c.c11 * v.y + c.c21 * v.z,
              c.c02 * v.x + c.c12 * v.y + c.c22 * v.z};
}
// c_bn^T . v and c_bn . v without forming the matrix: the ZYX dcm is Rx(roll) Ry(pitch) Rz(yaw),
// so each product is three planar rotations (12 multiply-adds instead of 16 + 9).  Same value as
// dcm_from_sincos + mul / mul_t up to rounding.
B2_DEV Vec3 rot_b2n(const SinCos3& t, const Vec3& v) {   // c^T . v
  // undo roll (about x)
  const double y1 = t.cr * v.y - t.sr * v.z;
  const double z1 = t.sr * v.y + t.cr * v.z;
  // undo pitch (about y)
  const double x2 = t.cp * v.x + t.sp * z1;
  const double z2 = -t.sp * v.x + t.cp * z1;
  // undo yaw (about z)
  return Vec3{t.cy * x2 - t.sy * y1, t.sy * x2 + t.cy * y1, z2};
}
B2_DEV Vec3 rot_n2b(const SinCos3& t, const Vec3& v) {   // c . v
  const double x1 = t.cy * v.x + t.sy * v.y;
  const double y1 = -t.sy * v.x + t.cy * v.y;
  const double x2 = t.cp * x1 - t.sp * v.z;
  const double z2 = t.sp * x1 + t.cp * v.z;
  return Vec3{x2, t.cr * y1 + t.sr * z2, -t.sr * y1 + t.cr * z2};
}

// attitude.cross3: attitude.py:758-770
B2_DEV Vec3 cross3(const Vec3& a, const Vec3& b) {
  return Vec3{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

// geoparams.geo_param: geoparams.py:25-53, given sin/cos of the latitude
struct GeoParam {
  double rm, rn, g, sl, cl;
};
B2_DEV GeoParam geo_param_sc(double sl, double cl, double h) {
  GeoParam p;
  p.sl = sl;
  p.cl = cl;
  const double sl_sqr = p.sl * p.sl;
  const double q = 1.0 - kESqr * sl_sqr;       // in [0.9933, 1]: no special cases
  const double inv_sq = rsqrt_nr(q);           // 1/sqrt(q): rm, rn and g only need the reciprocal root
  p.rm = ((kRe * (1 - kESqr)) * inv_sq) * (inv_sq * inv_sq);
  p.rn = kRe * inv_sq;
  const double g1 = kNormalGravity * (1 + kGravK * sl_sqr) * inv_sq;
  // (the reference divides 3 h^2 by Re twice, geoparams.py:52; one multiply by the constant 1 / Re^2
  // differs from that by an ulp of a 1e-9 g term and keeps two divisions out of the step's chain)
  p.g = g1 * (1.0 - (2.0 / kRe) * (1.0 + kFlat + kGravM - 2.0 * kFlat * sl_sqr) * h +
              (3.0 * h * h) * (1.0 / (kRe * kRe)));
  return p;
}
B2_DEV GeoParam geo_param(double lat, double h) {
  double sl, cl;
  sincos_angle(lat, &sl, &cl);
  return geo_param_sc(sl, cl, h);
}

// geoparams.lla2ecef: geoparams.py:70-87
B2_DEV Vec3 lla2ecef(double lat, double lon, double alt) {
  double sl, cl, so, co;
  sincos_angle(lat, &sl, &cl);
  sincos_angle(lon, &so, &co);
  const double r = kRe / sqrt(1.0 - kESqr * sl * sl);
  const double rho = (r + alt) * cl;
  return Vec3{rho * co, rho * so, (r * (1.0 - kESqr) + alt) * sl};
}

// attitude.angle_range_pi: attitude.py:799-812 (python float % : result has the sign of 2pi)
B2_DEV double angle_range_pi(double x) {
  double m = fmod(x, kTwoPi);
  if (m < 0.0) m += kTwoPi;
  if (m > kPi) m -= kTwoPi;
  return m;
}

// The navigation state of one Monte-Carlo run.
struct NavState {
  double yaw, pitch, roll;
  SinCos3 sc;  // sin/cos of (yaw, pitch, roll): euler2dcm(att[i]) of step i IS the
               // cos/sin euler_update_zyx needs at step i+1, so it is computed once
  double sl, cl;  // sin/cos of the latitude (ref_frame 0): geo_param of the NEXT step
  Vec3 vel_b;  // body velocity   (ref_frame 1 state)
  Vec3 vel;    // NED velocity    (ref_frame 0 state; ref_frame 1 output)
  Vec3 pos;    // ECEF-offset xyz (ref_frame 1) or lat, lon, alt (ref_frame 0)
  double g;    // gravity: geo_param(r0) or the ini override
  bool fixed_g;  // false: ref_frame 0 without override -> geo_param(pos) every step
  double icp;  // dt / cos(pitch), refreshed with the cosine (phi_dot = t / cos(pitch), attitude.py:693)
};

// ---- the incremental step --------------------------------------------------------------------
// Between two exact evaluations the sin/cos of an Euler angle (and of the latitude) are advanced by
// the angle-addition identity with the Taylor series of the increment d = rate * dt:
//     sin(a + d) = s + (s (cos d - 1) + c sin d),   cos(a + d) = c + (c (cos d - 1) - s sin d).
// |d| <= kRotMax = 2^-5 rad per step (179 deg/s at 100 Hz): the truncation error is below
// d^9/9! = 8e-20 (sin) and d^8/8! = 2.3e-17 (cos), the rounding one ulp of the increment per step.
// Every kResync steps -- and whenever an increment is larger than that, the pitch reflects, or the
// state is not finite -- the exact path (Cody-Waite sincos of the stored angle, as before) takes
// over, so the drift is bounded by kResync roundings (~7e-15) whatever the length of the series.
// What it buys: the loop-carried chain sincos(angle) -> rate -> angle -> sincos shrinks from about
// 250 cycles (reduction, two degree-6 polynomials, quadrant selects, a division) to about 80, and a
// step from 90 + 8 FP64 instructions of trigonometry to 39 + 5.
constexpr double kRotMax = 0.03125;
constexpr double kLatRotMax = 0.0009765625;   // 2^-10: the latitude moves ~1e-8 rad per step
constexpr int kResync = 64;

// ---- the speculative block ---------------------------------------------------------------------------
// Steps with SPEC = true (below) have no exact-path branch, so kSpecBlock of them unroll into one basic
// block and the scheduler overlaps the next step's rate products with the tail of the previous one.  If
// any lane of the warp needed the exact path (rare: an increment above kRotMax, a pitch reflection, a NaN)
// the warp restores the state saved before the block and redoes it step by step; every step computes the
// same numbers either way.  mc_spec_kernel.cuh, mc_av_kernel.cuh's attitude warp and the host test
// (tools/step_host.cu) all run spec_block.
constexpr int kSpecBlock = 4;
static_assert(kResync % kSpecBlock == 0, "a time-based re-evaluation falls on a block's last step");

// any lane of the warp; on the host (tools/step_host.cu) one lane is the warp
B2_DEV bool warp_any(bool x) {
#ifdef __CUDA_ARCH__
  return __any_sync(0xffffffffu, x);
#else
  return x;
#endif
}

// One block of kSpecBlock steps of state s.  With `speculate`: save s in `saved` (the caller keeps it in
// registers or shared memory), run spec(k) -- step k without the exact path, returning whether it was due --
// for k = 0 .. kSpecBlock - 1, vote, and on a cold vote restore s and run exact(k) for every k.  Without it:
// exact(k) at once.  Returns whether the block was run by exact().
#ifdef B2INS_HOST_TEST
#pragma nv_exec_check_disable   // the host test passes host lambdas
#endif
template <class State, class Spec, class Exact>
B2_DEV bool spec_block(bool speculate, State& s, State& saved, Spec&& spec, Exact&& exact) {
  bool redo = !speculate;
  if (speculate) {
    saved = s;
    bool cold = false;
#pragma unroll
    for (int k = 0; k < kSpecBlock; ++k) cold |= spec(k);
    redo = warp_any(cold);
    if (__builtin_expect(redo, 0)) s = saved;
  }
  if (redo) {
#pragma unroll 1
    for (int k = 0; k < kSpecBlock; ++k) exact(k);
  }
  return redo;
}

B2_DEV void rot_small(double& s, double& c, double d) {
  const double z = d * d;
  double ps = b2_fma(z, -1.98412698412698412698e-04, 8.33333333333333333333e-03);
  ps = b2_fma(z, ps, -1.66666666666666666667e-01);
  const double sd = b2_fma(d * z, ps, d);                 // sin d
  double pc = b2_fma(z, -1.38888888888888888889e-03, 4.16666666666666666667e-02);
  pc = b2_fma(z, pc, -0.5);
  const double cm1 = z * pc;                              // cos d - 1
  const double s2 = b2_fma(s, cm1, b2_fma(c, sd, s));
  const double c2 = b2_fma(c, cm1, b2_fma(-s, sd, c));
  s = s2;
  c = c2;
}
// |d| <= 2^-10: two terms each (d^5/120 < 8e-18, d^6/720 < 2e-21)
B2_DEV void rot_tiny(double& s, double& c, double d) {
  const double z = d * d;
  const double sd = b2_fma(d * z, -1.66666666666666666667e-01, d);
  const double cm1 = z * b2_fma(z, 4.16666666666666666667e-02, -0.5);
  const double s2 = b2_fma(s, cm1, b2_fma(c, sd, s));
  const double c2 = b2_fma(c, cm1, b2_fma(-s, sd, c));
  s = s2;
  c = c2;
}
// ONE +-2 pi wrap (attitude.py:712-720).  The fast step wraps yaw and roll only when it
// re-evaluates exactly (every kResync steps; they stay within +-(pi + kResync kRotMax) in between,
// and sin/cos do not notice); outputs are wrapped when they are written.
B2_DEV double wrap_once(double y) {
  return (y > kPi) ? (y - kTwoPi) : ((y < -kPi) ? (y + kTwoPi) : y);
}

// Refresh the cached sin/cos after the angles (and the latitude) moved.
// SPLIT (lane groups of >= 4 lanes): the state is replicated across the group, so the
// three (four with the latitude) independent sincos evaluations are spread over the lanes
// of each 4-lane subgroup -- lane role q evaluates angle q -- and exchanged by shuffles:
// one sincos worth of instruction issue instead of three or four.
template <int RF, bool SPLIT>
B2_DEV void refresh_trig(NavState& s, int role) {
  if (!SPLIT) {
    s.sc = sincos3(s.yaw, s.pitch, s.roll);
    if (RF == 0) sincos_angle(s.pos.x, &s.sl, &s.cl);
  } else {
    double a = s.roll;
    if (role == 0) a = s.yaw;
    if (role == 1) a = s.pitch;
    if (RF == 0 && role == 3) a = s.pos.x;
    double sv, cv;
    sincos_angle(a, &sv, &cv);
#ifdef __CUDA_ARCH__
    s.sc.sy = __shfl_sync(0xffffffffu, sv, 0, 4);
    s.sc.cy = __shfl_sync(0xffffffffu, cv, 0, 4);
    s.sc.sp = __shfl_sync(0xffffffffu, sv, 1, 4);
    s.sc.cp = __shfl_sync(0xffffffffu, cv, 1, 4);
    s.sc.sr = __shfl_sync(0xffffffffu, sv, 2, 4);
    s.sc.cr = __shfl_sync(0xffffffffu, cv, 2, 4);
    if (RF == 0) {
      s.sl = __shfl_sync(0xffffffffu, sv, 3, 4);
      s.cl = __shfl_sync(0xffffffffu, cv, 3, 4);
    }
#endif
  }
}

// free_integration.py:96-102 / :126-132 -- sample 0
template <int RF>
B2_DEV void nav_init(NavState& s, const double* __restrict__ ini,
                                         int ini_rows, double dt) {
  const double lat = ini[0], lon = ini[1], alt = ini[2];
  s.vel_b = Vec3{ini[3], ini[4], ini[5]};
  s.yaw = ini[6];
  s.pitch = ini[7];
  s.roll = ini[8];
  s.sl = s.cl = 0.0;
  if (RF == 1) {
    s.pos = lla2ecef(lat, lon, alt);
    s.g = (ini_rows > 9) ? ini[9] : geo_param(lat, alt).g;  // free_integration.py:89-93
    s.fixed_g = true;
  } else {
    s.pos = Vec3{lat, lon, alt};
    s.fixed_g = ini_rows > 9;  // free_integration.py:143-146
    s.g = s.fixed_g ? ini[9] : 0.0;
  }
  refresh_trig<RF, false>(s, 0);
  s.icp = rcp_nr(s.sc.cp) * dt;
  const Dcm c = dcm_from_sincos(s.sc);
  s.vel = mul_t(c, s.vel_b);
}

// The cold path of a step: everything derived from the angles, evaluated exactly from the stored
// angles -- pitch reflection (attitude.py:703-710), ONE +-2 pi wrap of yaw and roll (:712-720), then
// euler2dcm's sin/cos (:361-371) and the latitude's.  No shuffles: lanes of different runs take it
// independently.
template <int RF>
B2_DEV void resync_exact(NavState& s) {
  double y0 = s.yaw, y1 = s.pitch, y2 = s.roll;
  const bool hi = y1 > kHalfPi, lo = y1 < -kHalfPi;
  y1 = hi ? (kPi - y1) : (lo ? (-kPi - y1) : y1);
  const bool flip = hi || lo;
  y0 = flip ? y0 + kPi : y0;
  y2 = flip ? y2 + kPi : y2;
  s.yaw = wrap_once(y0);
  s.pitch = y1;
  s.roll = wrap_once(y2);
  refresh_trig<RF, false>(s, 0);
}

// One step i-1 -> i with the measurements of sample i-1.
//
// odo = false: FreeIntegration.run (free_integration.py:104-116 / :133-172).
// odo = true : free_integration_odo (free_integration_odo.py:104-112 / :121-158): same attitude
//              recurrence, body velocity = [odometer, 0, 0]; the odometer sample rides in accel.x.
// resync: re-evaluate the trigonometry exactly after this step (time-based, the same for every lane
// group width: results do not depend on the launch shape).
// attitude.euler_update_zyx (attitude.py:679-721) is inlined: t tan(pitch) = (t / cos(pitch)) sin(pitch),
// the reciprocal cosine (times dt) kept with the state so that no division sits on the yaw/roll chain.
// ODO: 0 = free integration, 1 = odometer variant (compile-time: no branch inside the step's basic
// block), 2 = decided by odo_rt at run time
// SPEC (speculative): the step WITHOUT the exact-path branch -- straight-line code, so that several steps
// unroll into one basic block and the scheduler overlaps them.  Returns whether the exact path was due
// (an increment above kRotMax, a pitch reflection, a NaN); spec_block then restores the state it saved
// and redoes the steps with SPEC = false.  (SPEC = false returns the same flag, already handled.)
template <int RF, bool SPLIT, int ODO = 0, bool SPEC = false>
B2_DEV bool nav_step(NavState& s, const Vec3& gyro, const Vec3& accel, double dt, bool earth_rot, int role,
                     bool resync, bool odo_rt = false) {
  const bool odo = (ODO == 2) ? odo_rt : (ODO == 1);
  const Vec3 vel_old = s.vel;
  Vec3 w = gyro;          // the rate that drives the Euler angles (w_nb_b in ref_frame 0)
  Vec3 cgdt, wxv;         // ref_frame 1: c_bn.dot(g_n) dt and gyro x vel_b of step i-1
  Vec3 fa, cor;           // ref_frame 0: c_bn^T accel and the Coriolis term of step i-1
  double g = s.g, dlat = 0.0;
  if (RF == 1) {
    // free_integration.py:104-116; g_n = [0,0,g]: third column of the OLD dcm, from the old sin/cos
    const double gdt = s.g * dt;
    const double cpg = s.sc.cp * gdt;
    cgdt = Vec3{-s.sc.sp * gdt, cpg * s.sc.sr, cpg * s.sc.cr};
    wxv = cross3(gyro, s.vel_b);
  } else {
    // free_integration.py:133-172
    const GeoParam p = geo_param_sc(s.sl, s.cl, s.pos.z);
    const double rm_e = p.rm + s.pos.z;
    const double rn_e = p.rn + s.pos.z;
    g = s.fixed_g ? s.g : p.g;
    const double inv_rn = rcp_nr(rn_e), inv_rm = rcp_nr(rm_e), inv_cl = rcp_nr(p.cl);
    const Vec3 w_en{s.vel.y * inv_rn, -s.vel.x * inv_rm, -s.vel.y * p.sl * inv_cl * inv_rn};
    Vec3 w_ie{0.0, 0.0, 0.0};
    if (earth_rot) {
      w_ie.x = kWie * p.cl;
      w_ie.z = -kWie * p.sl;
    }
    const Vec3 w_sum{w_en.x + w_ie.x, w_en.y + w_ie.y, w_en.z + w_ie.z};
    const Vec3 cw = rot_n2b(s.sc, w_sum);   // c_bn of step i-1
    w = Vec3{gyro.x - cw.x, gyro.y - cw.y, gyro.z - cw.z};
    fa = rot_b2n(s.sc, accel);
    const Vec3 w2{2 * w_ie.x + w_en.x, 2 * w_ie.y + w_en.y, 2 * w_ie.z + w_en.z};
    cor = cross3(w2, s.vel);
    dlat = vel_old.x * inv_rm * dt;
    s.pos.x += dlat;
    s.pos.y += vel_old.y * inv_rn * inv_cl * dt;
    s.pos.z += (-vel_old.z) * dt;
  }
  // ---- Euler-angle increments (attitude.py:691-700) from the sin/cos of the current angles ----
  const double t = b2_fma(w.z, s.sc.cr, w.y * s.sc.sr);
  const double dy = t * s.icp;                                         // phi_dot dt (icp = dt / cos pitch)
  const double dp = b2_fma(w.y, s.sc.cr, -(w.z * s.sc.sr)) * dt;       // theta_dot dt
  const double dr = b2_fma(dy, s.sc.sp, w.x * dt);                     // psi_dot dt
  s.yaw += dy;
  s.pitch += dp;
  s.roll += dr;
  // not-(<=) so that a NaN takes the exact path too; there sincos_angle keeps it NaN, so that from this
  // sample on the run is NaN as in the reference
  const bool cold = resync | !(fabs(s.pitch) <= kHalfPi) | !(fabs(dy) <= kRotMax) |
                    !(fabs(dp) <= kRotMax) | !(fabs(dr) <= kRotMax) |
                    (RF == 0 && !(fabs(dlat) <= kLatRotMax));
  if (!SPLIT) {
    rot_small(s.sc.sy, s.sc.cy, dy);
    rot_small(s.sc.sp, s.sc.cp, dp);
    rot_small(s.sc.sr, s.sc.cr, dr);
    if (RF == 0) rot_tiny(s.sl, s.cl, dlat);
  } else {
    // the lanes of a 4-lane subgroup share the work: role q advances angle q (3: the latitude)
    double sv = s.sc.sr, cv = s.sc.cr, d = dr;
    if (role == 0) { sv = s.sc.sy; cv = s.sc.cy; d = dy; }
    if (role == 1) { sv = s.sc.sp; cv = s.sc.cp; d = dp; }
    if (RF == 0 && role == 3) { sv = s.sl; cv = s.cl; d = dlat; }
    rot_small(sv, cv, d);
#ifdef __CUDA_ARCH__
    s.sc.sy = __shfl_sync(0xffffffffu, sv, 0, 4);
    s.sc.cy = __shfl_sync(0xffffffffu, cv, 0, 4);
    s.sc.sp = __shfl_sync(0xffffffffu, sv, 1, 4);
    s.sc.cp = __shfl_sync(0xffffffffu, cv, 1, 4);
    s.sc.sr = __shfl_sync(0xffffffffu, sv, 2, 4);
    s.sc.cr = __shfl_sync(0xffffffffu, cv, 2, 4);
    if (RF == 0) {
      s.sl = __shfl_sync(0xffffffffu, sv, 3, 4);
      s.cl = __shfl_sync(0xffffffffu, cv, 3, 4);
    }
#endif
  }
  if (!SPEC) {
    if (__builtin_expect(cold, 0)) resync_exact<RF>(s);
  }
  s.icp = rcp_nr(s.sc.cp) * dt;
  // ---- velocity, position ------------------------------------------------------------------
  if (RF == 1) {
    if (odo) {
      s.vel_b = Vec3{accel.x, 0.0, 0.0};
    } else {
      s.vel_b.x = b2_fma(-wxv.x, dt, b2_fma(accel.x, dt, s.vel_b.x) + cgdt.x);
      s.vel_b.y = b2_fma(-wxv.y, dt, b2_fma(accel.y, dt, s.vel_b.y) + cgdt.y);
      s.vel_b.z = b2_fma(-wxv.z, dt, b2_fma(accel.z, dt, s.vel_b.z) + cgdt.z);
    }
    s.vel = rot_b2n(s.sc, s.vel_b);
    s.pos.x = b2_fma(vel_old.x, dt, s.pos.x);
    s.pos.y = b2_fma(vel_old.y, dt, s.pos.y);
    s.pos.z = b2_fma(vel_old.z, dt, s.pos.z);
  } else {
    if (odo) {
      s.vel = rot_b2n(s.sc, Vec3{accel.x, 0.0, 0.0});   // c_bn of step i
    } else {
      s.vel.x = b2_fma(fa.x - cor.x, dt, vel_old.x);
      s.vel.y = b2_fma(fa.y - cor.y, dt, vel_old.y);
      s.vel.z = b2_fma(fa.z + g - cor.z, dt, vel_old.z);
    }
    // vel_b[i] = c_bn(i).dot(vel[i]) (:172) is not an output of the plugin; not computed
  }
  return cold;
}

// ---- ref_frame 1, the step split in two (mc_av_kernel.cuh) ------------------------------------------
// In the virtual inertial frame the attitude recurrence does not depend on velocity or position
// (free_integration.py:104: euler_update_zyx(att[i-1], gyro[i-1], dt)), so one warp can run it ahead and
// hand the sin/cos of every step to a second warp that does velocity and position (:109-116).
struct AttState {
  double yaw, pitch, roll;
  SinCos3 sc;
  double icp;   // dt / cos(pitch)
};

// the exact path of att_step (resync_exact on the attitude); icp is the caller's
B2_DEV void att_exact(AttState& s) {
  NavState n;            // the exact path works on the full state type
  n.yaw = s.yaw; n.pitch = s.pitch; n.roll = s.roll;
  n.pos = Vec3{0.0, 0.0, 0.0};
  resync_exact<1>(n);
  s.yaw = n.yaw; s.pitch = n.pitch; s.roll = n.roll;
  s.sc = n.sc;
}

// attitude.euler_update_zyx + euler2dcm's sin/cos for the new angles: the attitude half of nav_step<1>
// SPEC: without the exact-path branch, returns whether it was due (see nav_step)
template <bool SPEC = false>
B2_DEV bool att_step(AttState& s, const Vec3& w, double dt, bool resync) {
  const double t = b2_fma(w.z, s.sc.cr, w.y * s.sc.sr);
  const double dy = t * s.icp;
  const double dp = b2_fma(w.y, s.sc.cr, -(w.z * s.sc.sr)) * dt;
  const double dr = b2_fma(dy, s.sc.sp, w.x * dt);
  s.yaw += dy;
  s.pitch += dp;
  s.roll += dr;
  const bool cold = resync | !(fabs(s.pitch) <= kHalfPi) | !(fabs(dy) <= kRotMax) |
                    !(fabs(dp) <= kRotMax) | !(fabs(dr) <= kRotMax);
  rot_small(s.sc.sy, s.sc.cy, dy);
  rot_small(s.sc.sp, s.sc.cp, dp);
  rot_small(s.sc.sr, s.sc.cr, dr);
  if (!SPEC && __builtin_expect(cold, 0)) att_exact(s);
  s.icp = rcp_nr(s.sc.cp) * dt;
  return cold;
}

struct VelState {
  Vec3 vel_b, vel, pos;
  double gdt;   // g dt
};

// free_integration.py:109-116 with the sin/cos of step i-1 (old) and step i (now)
B2_DEV void vel_step(VelState& s, const Vec3& gyro, const Vec3& accel, const SinCos3& old, const SinCos3& now,
                     double dt) {
  const double cpg = old.cp * s.gdt;
  const Vec3 cgdt{-old.sp * s.gdt, cpg * old.sr, cpg * old.cr};
  const Vec3 wxv = cross3(gyro, s.vel_b);
  const Vec3 vel_old = s.vel;
  s.vel_b.x = b2_fma(-wxv.x, dt, b2_fma(accel.x, dt, s.vel_b.x) + cgdt.x);
  s.vel_b.y = b2_fma(-wxv.y, dt, b2_fma(accel.y, dt, s.vel_b.y) + cgdt.y);
  s.vel_b.z = b2_fma(-wxv.z, dt, b2_fma(accel.z, dt, s.vel_b.z) + cgdt.z);
  s.vel = rot_b2n(now, s.vel_b);
  s.pos.x = b2_fma(vel_old.x, dt, s.pos.x);
  s.pos.y = b2_fma(vel_old.y, dt, s.pos.y);
  s.pos.z = b2_fma(vel_old.z, dt, s.pos.z);
}

}  // namespace b2ins
