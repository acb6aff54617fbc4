// Host build of the strapdown step the kernels run (csrc/mech.cuh with B2INS_HOST_TEST): one run of
// free integration on supplied gyro/accel, for the CPU-side check against the oracle
// (tests/test_cpu_step.py), step by step or in the speculative blocks of the fused kernels
// (tests/test_cpu_exact_path.py).  Test tooling; not part of libb2ins.so.
//   nvcc -O2 -std=c++17 -shared -Xcompiler -fPIC -DB2INS_HOST_TEST -o tools/libstep_host.so tools/step_host.cu
#include "../gnss_ins_sim_b200/csrc/mech.cuh"

using namespace b2ins;

template <int RF>
static void run(int64_t n, double dt, int earth_rot, int odo, const double* gyro, const double* accel,
                const double* ini, int ini_rows, int resync_every, double* att, double* pos, double* vel) {
  NavState st;
  nav_init<RF>(st, ini, ini_rows, dt);
  for (int64_t i = 0; i < n; ++i) {
    att[i * 3 + 0] = i ? wrap_once(st.yaw) : st.yaw;
    att[i * 3 + 1] = st.pitch;
    att[i * 3 + 2] = i ? wrap_once(st.roll) : st.roll;
    pos[i * 3 + 0] = st.pos.x; pos[i * 3 + 1] = st.pos.y; pos[i * 3 + 2] = st.pos.z;
    vel[i * 3 + 0] = st.vel.x; vel[i * 3 + 1] = st.vel.y; vel[i * 3 + 2] = st.vel.z;
    if (i + 1 == n) break;
    const Vec3 w{gyro[i * 3], gyro[i * 3 + 1], gyro[i * 3 + 2]};
    const Vec3 f{accel[i * 3], accel[i * 3 + 1], accel[i * 3 + 2]};
    const bool resync = resync_every > 0 ? ((i + 1) % resync_every) == 0 : false;
    if (odo)
      nav_step<RF, false, 1>(st, w, f, dt, earth_rot != 0, 0, resync);
    else
      nav_step<RF, false, 0>(st, w, f, dt, earth_rot != 0, 0, resync);
  }
}

extern "C" int step_host_free_integration(int ref_frame, int64_t n, double fs, int earth_rot, int odo,
                                          const double* gyro, const double* accel, const double* ini,
                                          int ini_rows, int resync_every, double* att, double* pos,
                                          double* vel) {
  if (ref_frame == 1)
    run<1>(n, 1.0 / fs, earth_rot, odo, gyro, accel, ini, ini_rows, resync_every, att, pos, vel);
  else
    run<0>(n, 1.0 / fs, earth_rot, odo, gyro, accel, ini, ini_rows, resync_every, att, pos, vel);
  return 0;
}
extern "C" int step_host_resync_default(void) { return kResync; }

// ---- the speculative blocks of the fused Monte-Carlo kernels, for one run (one lane of a warp) ----------
// Steps are taken in blocks of kSpecBlock from step 0 while a whole block is left, the rest one by one, with the
// time-based re-evaluation after every kResync-th sample, as the kernels do.  A block is the kernels' own
// spec_block (mech.cuh); what is here is what the kernels do around it.  The rows of a block are written once
// it has settled: what the kernels' end state and ring hold, not their (non-speculative) history path.

static void put_row(double* o, int64_t i, double x, double y, double z) {
  o[i * 3 + 0] = x; o[i * 3 + 1] = y; o[i * 3 + 2] = z;
}

// mc_av_kernel.cuh (ref_frame 1): warp A runs att_step<true> in speculative blocks, redone with att_step<false>;
// after a warm block whose last sample is a multiple of kResync, att_exact and the new 1/cos replace the last
// step's sin/cos.  Warp V then runs vel_step on the sin/cos before and after every step (the ring).
extern "C" int step_host_av_blocks(int64_t n, double fs, const double* gyro, const double* accel, const double* ini,
                                   int ini_rows, double* att, double* pos, double* vel) {
  const double dt = 1.0 / fs;
  NavState st0;
  nav_init<1>(st0, ini, ini_rows, dt);
  AttState a;
  a.yaw = st0.yaw; a.pitch = st0.pitch; a.roll = st0.roll;
  a.sc = st0.sc;
  a.icp = st0.icp;
  VelState v;
  v.vel_b = st0.vel_b; v.vel = st0.vel; v.pos = st0.pos;
  v.gdt = st0.g * dt;
  SinCos3 old = st0.sc;
  if (n <= 0) return 0;
  put_row(att, 0, a.yaw, a.pitch, a.roll);
  put_row(pos, 0, v.pos.x, v.pos.y, v.pos.z);
  put_row(vel, 0, v.vel.x, v.vel.y, v.vel.z);
  for (int64_t s = 0; s < n - 1;) {
    const int len = (s + kSpecBlock <= n - 1) ? kSpecBlock : 1;
    SinCos3 ring[kSpecBlock];
    double ang[kSpecBlock][3];
    auto keep = [&](int k) {
      ring[k] = a.sc;
      ang[k][0] = a.yaw; ang[k][1] = a.pitch; ang[k][2] = a.roll;
    };
    auto w_of = [&](int64_t i) { return Vec3{gyro[i * 3], gyro[i * 3 + 1], gyro[i * 3 + 2]}; };
    if (len == kSpecBlock) {
      AttState saved;
      const bool redone = spec_block(true, a, saved, [&](int k) {
        const bool cold = att_step<true>(a, w_of(s + k), dt, false);
        keep(k);
        return cold;
      }, [&](int k) {
        att_step(a, w_of(s + k), dt, ((s + k + 1) & (kResync - 1)) == 0);
        keep(k);
      });
      if (!redone && ((s + kSpecBlock) & (kResync - 1)) == 0) {
        att_exact(a);
        a.icp = rcp_nr(a.sc.cp) * dt;
        keep(kSpecBlock - 1);
      }
    } else {
      att_step(a, w_of(s), dt, ((s + 1) & (kResync - 1)) == 0);
      keep(0);
    }
    for (int k = 0; k < len; ++k) {
      const int64_t i = s + k;
      const Vec3 f{accel[i * 3], accel[i * 3 + 1], accel[i * 3 + 2]};
      vel_step(v, w_of(i), f, old, ring[k], dt);
      old = ring[k];
      put_row(att, i + 1, wrap_once(ang[k][0]), ang[k][1], wrap_once(ang[k][2]));
      put_row(pos, i + 1, v.pos.x, v.pos.y, v.pos.z);
      put_row(vel, i + 1, v.vel.x, v.vel.y, v.vel.z);
    }
    s += len;
  }
  return 0;
}

// mc_spec_kernel.cuh: nav_step<RF, false, ODO, true> in speculative blocks, redone step by step with the exact
// path; a block that holds the time-based re-evaluation is not speculated.  (The kernel runs free integration only; the odometer variant shares the step and is checked too.)
template <int RF, int ODO>
static void spec_blocks(int64_t n, double dt, int earth_rot, const double* gyro, const double* accel,
                        const double* ini, int ini_rows, double* att, double* pos, double* vel) {
  NavState st;
  nav_init<RF>(st, ini, ini_rows, dt);
  if (n <= 0) return;
  put_row(att, 0, st.yaw, st.pitch, st.roll);
  put_row(pos, 0, st.pos.x, st.pos.y, st.pos.z);
  put_row(vel, 0, st.vel.x, st.vel.y, st.vel.z);
  for (int64_t s = 0; s < n - 1;) {
    const int len = (s + kSpecBlock <= n - 1) ? kSpecBlock : 1;
    NavState after[kSpecBlock];
    auto one = [&](int64_t i, bool spec) {
      const Vec3 w{gyro[i * 3], gyro[i * 3 + 1], gyro[i * 3 + 2]};
      const Vec3 f{accel[i * 3], accel[i * 3 + 1], accel[i * 3 + 2]};
      if (spec) return nav_step<RF, false, ODO, true>(st, w, f, dt, earth_rot != 0, 0, false);
      return nav_step<RF, false, ODO>(st, w, f, dt, earth_rot != 0, 0, ((i + 1) & (kResync - 1)) == 0);
    };
    if (len == kSpecBlock) {
      NavState saved;
      const bool speculate = (s & (kResync - 1)) + kSpecBlock < kResync;
      spec_block(speculate, st, saved, [&](int k) {
        const bool cold = one(s + k, true);
        after[k] = st;
        return cold;
      }, [&](int k) {
        one(s + k, false);
        after[k] = st;
      });
    } else {
      one(s, false);
      after[0] = st;
    }
    for (int k = 0; k < len; ++k) {
      const NavState& t = after[k];
      put_row(att, s + k + 1, wrap_once(t.yaw), t.pitch, wrap_once(t.roll));
      put_row(pos, s + k + 1, t.pos.x, t.pos.y, t.pos.z);
      put_row(vel, s + k + 1, t.vel.x, t.vel.y, t.vel.z);
    }
    s += len;
  }
}

extern "C" int step_host_spec_blocks(int ref_frame, int64_t n, double fs, int earth_rot, int odo, const double* gyro,
                                     const double* accel, const double* ini, int ini_rows, double* att, double* pos,
                                     double* vel) {
  const double dt = 1.0 / fs;
  if (ref_frame == 1)
    (odo ? spec_blocks<1, 1> : spec_blocks<1, 0>)(n, dt, earth_rot, gyro, accel, ini, ini_rows, att, pos, vel);
  else
    (odo ? spec_blocks<0, 1> : spec_blocks<0, 0>)(n, dt, earth_rot, gyro, accel, ini, ini_rows, att, pos, vel);
  return 0;
}
