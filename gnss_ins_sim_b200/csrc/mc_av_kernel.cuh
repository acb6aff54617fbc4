// K12, ref_frame 1, few runs: the STEP ITSELF split over two warps.
//
// With 1000 runs an H100 has about one integrator warp per SM, and that warp's step is ~120 instructions,
// most of them FP64, on dependency chains: it is bound by the dependent-issue latency of one warp (DESIGN.md 3.2).
// In the virtual inertial frame the attitude recurrence does not read velocity or position
// (free_integration.py:104), so it runs ahead in its own warp and hands the sin/cos of every step
// through a shared-memory ring to a second warp that does velocity and position (:109-116):
//
//   producers (one job = a channel of four runs x 8 samples)  --slots-->  A: rates, three rotations, 1/cos
//                                                              \--slots-->  V: c_bn g, w x v, v_b, v = c_bn^T v_b, pos   <--ring-- A
//
// One named barrier per round of kAvRound samples couples the three stages: in interval i the
// producers fill round i, A integrates round i-1, V round i-2 (slots triple-buffered, the ring
// double-buffered).  A is the critical path; the warp placement is in the
// role tables below.
#pragma once
#include "mc_spec_kernel.cuh"

namespace b2ins {

constexpr int kAvRound = 8;
// A producer warp always works on four runs x the eight samples of a round (one Box-Muller pass per round,
// its own Gauss-Markov carry): six of them with groups of 8 lanes (four runs per CTA), twelve with groups
// of 4 (eight runs per CTA: two producers per channel, one for each half of the runs).
template <int G>
struct AvShape {
  static constexpr int kHalves = (32 / G) / 4;
  static constexpr int kProd = 6 * kHalves;
  static constexpr int kWarps = (G == 4) ? 16 : 12;
  static constexpr int kSync = 32 * (2 + kProd);      // A + V + producers
};
// role of warp w (it runs on sub-partition w % 4): -1 = A, -2 = V, -3 = leaves at once, else producer index.
// A (warp 0) is the critical path: alone on sub-partition 0 with groups of 8, with ONE producer (warp 4)
// with groups of 4; V, idle more than half of the time, shares sub-partition 1 with two / three producers.
__device__ constexpr int kAvRole8[12] = {-1, -2, 0, 1, -3, 2, 3, 4, -3, 5, -3, -3};
__device__ constexpr int kAvRole4[16] = {-1, -2, 0, 1, 2, 3, 4, 5, -3, 6, 7, 8, -3, 9, 10, 11};

template <int G>
struct AvSmem {
  alignas(128) double gyro[kStagesFast][kTile * 3];
  alignas(128) double accel[kStagesFast][kTile * 3];
  alignas(16) SampleSlot slot[3][kAvRound / G][32];
  alignas(16) double ring[2][kAvRound][32 / G][6];       // sin/cos after every step, per run of the CTA
  alignas(8) uint64_t full[kStagesFast];
  alignas(8) uint64_t empty[kStagesFast];
};

template <int G>
__global__ void __launch_bounds__(AvShape<G>::kWarps * 32, 1) mc_av_kernel(const __grid_constant__ McParams p) {
  static_assert(G == 4 || G == 8, "groups of 4 or 8 lanes");
  constexpr int kRunsPerCta = 32 / G;
  constexpr int kProd = AvShape<G>::kProd;
  constexpr int kAvSync = AvShape<G>::kSync;
  __shared__ AvSmem<G> sm;
  const int lane = threadIdx.x & 31;
  const int pwarp = threadIdx.x >> 5;
  const int role_w = (G == 4) ? kAvRole4[pwarp] : kAvRole8[pwarp];
  const bool is_a = role_w == -1, is_v = role_w == -2, is_p = role_w >= 0;
  const int pp = is_p ? role_w : 0;                        // producer index: channel pp % 6, run half pp / 6
  // A and V: G lanes per run.  Producers: eight lanes per run (the samples of a round), four runs.
  const int j = is_p ? (lane & 7) : lane % G;
  const int grp = is_p ? (pp / 6) * 4 + (lane >> 3) : lane / G;      // run within the CTA
  const int64_t run_raw = static_cast<int64_t>(blockIdx.x) * kRunsPerCta + grp;
  const bool active = run_raw < p.runs;
  const int64_t run = active ? run_raw : p.runs - 1;
  const int64_t grun = p.run_offset + run;
  const uint32_t run_lo = static_cast<uint32_t>(grun), run_hi = static_cast<uint32_t>(grun >> 32);
  const bool dump = active && run < p.dump_runs;
  const bool warp_dumps = __any_sync(0xffffffffu, dump);
  const int64_t num_tiles = (p.n + kTile - 1) / kTile;
  const int issuer = 2 * 32;                               // lane 0 of the first producer warp
  auto stage_sync = [&]() { asm volatile("bar.sync 1, %0;" ::"n"(kAvSync) : "memory"); };

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStagesFast; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], kProd);
    }
    mbar_fence_init();
  }
  __syncthreads();
  if (!is_a && !is_v && !is_p) return;                     // the spare warps
  // rounds of the whole series: tiles are whole rounds (kTile % kAvRound == 0), the last may be short
  const int64_t rounds = (p.n + kAvRound - 1) / kAvRound;

  if (is_p) {
    // =============================== producer: channel pp =========================================
    if (threadIdx.x == issuer)
      for (int s = 0; s < kStagesFast && s < num_tiles; ++s) spec_issue_tile(sm, p, s, s);
    const int c = pp % 6, ax = c % 3;
    const bool is_acc = c < 3;
    const TriadNoise& e = is_acc ? p.accel : p.gyro;
    double carry = 0.0;
    const double apj = ipow(e.gm_a[ax], j), aG = ipow(e.gm_a[ax], kAvRound);
    double phase[3] = {0.0, 0.0, 0.0};
    if (p.gyro.vib_type == 2) {
#pragma unroll
      for (int k = 0; k < 3; ++k)
        phase[k] = (uniform01(0xFFFFFFFFu, kDrawPhase + k, run_lo, run_hi, p.k0, p.k1) * 2.0) * kPi;
    }
    const bool any_vib = (p.accel.vib_type | p.gyro.vib_type) != 0;
    for (int64_t i = 0; i < rounds + 2; ++i) {
      if (i < rounds) {
        const int64_t r0 = i * kAvRound;                   // first sample of the round
        const int64_t tile = r0 / kTile;
        const int s = static_cast<int>(tile % kStagesFast);
        const int base = static_cast<int>(r0 - tile * kTile);
        const int cnt = static_cast<int>(min64(kTile, p.n - tile * kTile));
        if (base == 0) {
          // refill the stage the PREVIOUS tile used, then wait for this tile's data
          if (threadIdx.x == issuer && tile >= 1 && tile - 1 + kStagesFast < num_tiles) {
            const int sp = static_cast<int>((tile - 1) % kStagesFast);
            mbar_wait(&sm.empty[sp], static_cast<uint32_t>(((tile - 1) / kStagesFast) & 1));
            spec_issue_tile(sm, p, tile - 1 + kStagesFast, sp);
          }
          mbar_wait(&sm.full[s], static_cast<uint32_t>((tile / kStagesFast) & 1));
        }
        const int buf = static_cast<int>(i % 3);
        {
          const int tj = base + j;
          const int64_t t = tile * kTile + tj;
          const bool live = tj < cnt;
          Normal2 z{0.0, 0.0};
          double m = 0.0;
          if (live) {
            z = normal_pair(static_cast<uint32_t>(t), c, run_lo, run_hi, p.k0, p.k1);
            const double ref = is_acc ? sm.accel[s][tj * 3 + ax] : sm.gyro[s][tj * 3 + ax];
            m = (ref + e.b[ax]) + e.w[ax] * z.z1;
            if (any_vib)
              m += vib_term(e, ax, is_acc ? 0 : 1, static_cast<uint32_t>(t), run_lo, run_hi, p.k0, p.k1, run, phase);
          }
          const double d = gm_block<kAvRound>(e.gm_b[ax] * z.z0, e.gm_a[ax], apj, aG, j, carry);
          m += d + e.wd[ax] * z.z0;
          int64_t row;
          if (warp_dumps && dump && live && p.out_gyro && dump_row(p, t, &row))
            (is_acc ? p.out_accel : p.out_gyro)[run * p.osr + row * p.ost + ax * p.osc] = m;
          // sample j of run grp, where the consumers (G lanes per run, passes of G samples) look for it
          SampleSlot& mine = sm.slot[buf][j / G][grp * G + (j % G)];
          if (is_acc) mine.a[ax] = m; else mine.g[ax] = m;
        }
        if (base + kAvRound >= cnt) {                      // last round of the tile: release the stage
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm.empty[s]);
        }
      }
      if (i <= rounds) stage_sync();     // intervals 0 .. rounds end in a barrier; the last one is V's alone
    }
    return;
  }

  // initial state (both A and V derive what they need from it)
  NavState st0;
  {
    const int64_t irun = p.ini_offset + run;
    const int64_t set = (irun < p.ini_sets) ? irun : 0;  // free_integration.py:85-87
    nav_init<1>(st0, p.ini + set * p.ini_rows, p.ini_rows, p.dt);
  }

  if (is_a) {
    // ================================= A: attitude =================================================
    AttState a;
    a.yaw = st0.yaw; a.pitch = st0.pitch; a.roll = st0.roll;
    a.sc = st0.sc;
    a.icp = st0.icp;
    if (dump && j == 0 && p.out_att) {
      const int64_t o = run * p.osr;
      p.out_att[o] = a.yaw;
      p.out_att[o + p.osc] = a.pitch;
      p.out_att[o + 2 * p.osc] = a.roll;
      if (p.out_quat) write_quat(p.out_quat + run * p.dump_rows * 4, a.yaw, a.pitch, a.roll);
    }
    for (int64_t i = 0; i < rounds + 2; ++i) {
      if (i >= 1 && i <= rounds) {
        const int64_t r0 = (i - 1) * kAvRound;
        const int sbuf = static_cast<int>((i - 1) % 3), rbuf = static_cast<int>((i - 1) & 1);
        // samples of this round that are followed by a step (the last sample of the series is not)
        const int kmax = static_cast<int>(min64(kAvRound, p.n - 1 - r0));
        auto a_step = [&](int k) {                        // one step with the exact path and the history rows
          const SampleSlot& sl = sm.slot[sbuf][k / G][lane - j + (k % G)];
          const Vec3 w{sl.g[0], sl.g[1], sl.g[2]};
          att_step(a, w, p.dt, ((r0 + k + 1) & (kResync - 1)) == 0);
          if (j == 0) {
            double* o = sm.ring[rbuf][k][grp];
            reinterpret_cast<double2*>(o)[0] = make_double2(a.sc.sy, a.sc.cy);
            reinterpret_cast<double2*>(o)[1] = make_double2(a.sc.sp, a.sc.cp);
            reinterpret_cast<double2*>(o)[2] = make_double2(a.sc.sr, a.sc.cr);
          }
          int64_t row;
          if (warp_dumps && dump && j == 0 && p.out_att && dump_row(p, r0 + k + 1, &row)) {
            const int64_t o = run * p.osr + row * p.ost;
            const double y = wrap_once(a.yaw), r = wrap_once(a.roll);
            p.out_att[o] = y;
            p.out_att[o + p.osc] = a.pitch;
            p.out_att[o + 2 * p.osc] = r;
            if (p.out_quat) write_quat(p.out_quat + (run * p.dump_rows + row) * 4, y, a.pitch, r);
          }
        };
        if (warp_dumps || kmax < kAvRound) {
#pragma unroll 1
          for (int k = 0; k < kmax; ++k) a_step(k);
        } else {
          // Blocks of four steps as ONE basic block without the exact-path branch (mc_spec_kernel.cuh has
          // the same scheme): the next step's loads and rate products overlap the tail of the previous
          // one.  A block that holds a time-based re-evaluation (1 of 16), or in which any lane needed
          // the exact path, is (re)done step by step from the saved state; the ring is overwritten with
          // the same or the corrected values before V sees it (V reads after the next barrier).
#pragma unroll 1
          for (int kb = 0; kb < kAvRound; kb += 4) {
            bool redo = ((r0 + kb) & (kResync - 1)) + 4 >= kResync;
            if (!redo) {
              const AttState saved = a;
              bool cold = false;
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                const SampleSlot& sl = sm.slot[sbuf][(kb + k) / G][lane - j + ((kb + k) % G)];
                const Vec3 w{sl.g[0], sl.g[1], sl.g[2]};
                cold |= att_step<true>(a, w, p.dt, false);
                if (j == 0) {
                  double* o = sm.ring[rbuf][kb + k][grp];
                  reinterpret_cast<double2*>(o)[0] = make_double2(a.sc.sy, a.sc.cy);
                  reinterpret_cast<double2*>(o)[1] = make_double2(a.sc.sp, a.sc.cp);
                  reinterpret_cast<double2*>(o)[2] = make_double2(a.sc.sr, a.sc.cr);
                }
              }
              redo = __any_sync(0xffffffffu, cold);
              if (__builtin_expect(redo, 0)) a = saved;
            }
            if (redo) {
#pragma unroll 1
              for (int k = 0; k < 4; ++k) a_step(kb + k);
            }
          }
        }
      }
      if (i <= rounds) stage_sync();
    }
    if (active && j == 0) {
      const double* r = p.ref_nav + (p.n - 1) * 9;
      if (p.end_err) {
        double* e = p.end_err + run * 9;
        e[0] = angle_range_pi(a.yaw - r[0]);
        e[1] = angle_range_pi(a.pitch - r[1]);
        e[2] = angle_range_pi(a.roll - r[2]);
      }
      if (p.end_state) {
        double* e = p.end_state + run * 9;
        e[0] = wrap_once(a.yaw); e[1] = a.pitch; e[2] = wrap_once(a.roll);
      }
    }
    return;
  }

  // =================================== V: velocity, position ========================================
  VelState v;
  v.vel_b = st0.vel_b;
  v.vel = st0.vel;
  v.pos = st0.pos;
  v.gdt = st0.g * p.dt;
  SinCos3 old = st0.sc;
  if (dump && j == 0 && p.out_att) {
    const int64_t o = run * p.osr;
    p.out_pos[o] = v.pos.x;
    p.out_pos[o + p.osc] = v.pos.y;
    p.out_pos[o + 2 * p.osc] = v.pos.z;
    p.out_vel[o] = v.vel.x;
    p.out_vel[o + p.osc] = v.vel.y;
    p.out_vel[o + 2 * p.osc] = v.vel.z;
  }
  for (int64_t i = 0; i < rounds + 2; ++i) {
    if (i >= 2) {
      const int64_t r0 = (i - 2) * kAvRound;
      const int sbuf = static_cast<int>((i - 2) % 3), rbuf = static_cast<int>((i - 2) & 1);
      const int kmax = static_cast<int>(min64(kAvRound, p.n - 1 - r0));
      auto v_step = [&](int k, bool hist) {
        const SampleSlot& sl = sm.slot[sbuf][k / G][lane - j + (k % G)];
        const Vec3 w{sl.g[0], sl.g[1], sl.g[2]};
        const Vec3 f{sl.a[0], sl.a[1], sl.a[2]};
        const double2* o = reinterpret_cast<const double2*>(sm.ring[rbuf][k][grp]);
        const double2 q0 = o[0], q1 = o[1], q2 = o[2];
        SinCos3 now;
        now.sy = q0.x; now.cy = q0.y; now.sp = q1.x; now.cp = q1.y; now.sr = q2.x; now.cr = q2.y;
        vel_step(v, w, f, old, now, p.dt);
        old = now;
        int64_t row;
        if (hist && dump && j == 0 && p.out_att && dump_row(p, r0 + k + 1, &row)) {
          const int64_t oo = run * p.osr + row * p.ost;
          p.out_pos[oo] = v.pos.x;
          p.out_pos[oo + p.osc] = v.pos.y;
          p.out_pos[oo + 2 * p.osc] = v.pos.z;
          p.out_vel[oo] = v.vel.x;
          p.out_vel[oo + p.osc] = v.vel.y;
          p.out_vel[oo + 2 * p.osc] = v.vel.z;
        }
      };
      if (warp_dumps || kmax < kAvRound) {
#pragma unroll 1
        for (int k = 0; k < kmax; ++k) v_step(k, true);
      } else {
#pragma unroll 1
        for (int kb = 0; kb < kAvRound; kb += 4) {
#pragma unroll
          for (int k = 0; k < 4; ++k) v_step(kb + k, false);
        }
      }
    }
    if (i <= rounds) stage_sync();        // V's last round follows the last barrier
  }
  if (active && j == 0) {
    const double* r = p.ref_nav + (p.n - 1) * 9;
    if (p.end_err) {
      double* e = p.end_err + run * 9;
      e[3] = v.pos.x - r[3];
      e[4] = v.pos.y - r[4];
      e[5] = v.pos.z - r[5];
      e[6] = v.vel.x - r[6];
      e[7] = v.vel.y - r[7];
      e[8] = v.vel.z - r[8];
    }
    if (p.end_state) {
      double* e = p.end_state + run * 9;
      e[3] = v.pos.x; e[4] = v.pos.y; e[5] = v.pos.z;
      e[6] = v.vel.x; e[7] = v.vel.y; e[8] = v.vel.z;
    }
  }
}

}  // namespace b2ins
