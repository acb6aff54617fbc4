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
// role tables below.  Phase clocks per role (tools/spec2_phase.py, one H100 SXM 80 GB at a 400 W power
// limit, 1000 runs, G = 4): A spends ~95 % of a round stepping and ~5 % at the barrier, V and the producers
// wait ~50 % and ~30 % of it.  So A's block is what a round costs: its slot loads are issued at the start
// of the block, and the time-based re-evaluation runs in a speculative block like the others.  The producers
// issue fewer instructions per round too (with groups of 4 one of them shares A's sub-partition).  Config 2:
// 0.170 -> 0.137 ms (0.160 with the lighter producers alone); 500 runs, G = 8: 0.142 -> 0.119 ms.
#pragma once
#include <type_traits>

#include "mc_spec_kernel.cuh"

namespace b2ins {

constexpr int kAvRound = 8;
static_assert(kAvRound % kSpecBlock == 0, "A's rounds are whole speculative blocks");
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

// Phase clocks (-DB2INS_PHASE_CLOCKS, tools/spec2_phase.py): g_phase_clocks[8] A stepping, [9] A at the
// barrier, [10] A's time-based re-evaluation after a warm block, [11] V stepping, [12] V at the barrier,
// [13] producers waiting for a tile, [14] producing, [15] producers at the barrier.  B2INS_MC_DEBUG idles
// the producers (1), A (2) or V (4).

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
  const McRun mr = mc_run(p, static_cast<int64_t>(blockIdx.x) * kRunsPerCta + grp);
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
#ifdef B2INS_PHASE_CLOCKS
  // isolation runs read slots or a ring nobody wrote: zeros keep A off the exact path
  if (p.debug) {
    for (int q = threadIdx.x; q < static_cast<int>(sizeof(sm.slot) / 8); q += blockDim.x)
      reinterpret_cast<double*>(sm.slot)[q] = 0.0;
    for (int q = threadIdx.x; q < static_cast<int>(sizeof(sm.ring) / 8); q += blockDim.x)
      reinterpret_cast<double*>(sm.ring)[q] = 0.0;
  }
#endif
  __syncthreads();
  if (!is_a && !is_v && !is_p) return;                     // the spare warps
  // rounds of the whole series: tiles are whole rounds (kTile % kAvRound == 0), the last may be short
  const int64_t rounds = (p.n + kAvRound - 1) / kAvRound;

  if (is_p) {
    // =============================== producer: channel pp =========================================
    if (threadIdx.x == issuer)
      for (int s = 0; s < kStagesFast && s < num_tiles; ++s) issue_tile<false, false>(sm, p, s, s);
    const int c = pp % 6, ax = c % 3;
    const bool is_acc = c < 3;
    const TriadNoise& e = is_acc ? p.accel : p.gyro;
    // The channel's error model in registers for the whole series: read in the round loop, every
    // coefficient is a parameter-space load indexed by the channel.
    const double eb = e.b[ax], ew = e.w[ax], ewd = e.wd[ax], ga = e.gm_a[ax], gb = e.gm_b[ax];
    double carry = 0.0;
    const double apj = ipow(ga, j), aG = ipow(ga, kAvRound);
    double phase[3] = {0.0, 0.0, 0.0};
    if (p.gyro.vib_type == 2) {
#pragma unroll
      for (int k = 0; k < 3; ++k)
        phase[k] = (uniform01(0xFFFFFFFFu, kDrawPhase + k, mr.lo, mr.hi, p.k0, p.k1) * 2.0) * kPi;
    }
    const bool any_vib = (p.accel.vib_type | p.gyro.vib_type) != 0;
    // This lane's sample (base + j) of the round in the trajectory tile of stage s is ref0[s kTile 3 +
    // 3 base]; its slot (sample j of run grp, where the consumers -- G lanes per run, passes of G
    // samples -- look for it) in slot set buf is out0[buf kSlotSet].
    const double* ref0 = (is_acc ? sm.accel[0] : sm.gyro[0]) + j * 3 + ax;
    SampleSlot& slot0 = sm.slot[0][j / G][grp * G + (j % G)];
    double* out0 = (is_acc ? slot0.a : slot0.g) + ax;
    constexpr int kSlotSet = static_cast<int>(sizeof(sm.slot[0]) / sizeof(double));
    const int nrounds = static_cast<int>(rounds);         // n < 2^32 (b2ins_api.cu)
    const int ntiles = static_cast<int>(num_tiles);
    // The round loop, with the history output and the vibration models compiled in (SLOW) or out: the
    // choice is made once per warp.  Tile, stage, parity and slot set advance by counting.
    auto produce = [&](auto slow) {
      constexpr bool kSlow = decltype(slow)::value;
      int tile = 0, s = 0, base = 0, ref_off = 0, out_off = 0;
      uint32_t parity = 0, t0 = 0;
      int cnt = static_cast<int>(min64(kTile, p.n));
      for (int i = 0; i < nrounds; ++i) {
        if (base == 0) refill_and_wait<false, false>(sm, p, threadIdx.x == issuer, tile, ntiles, s, parity, 13);
        B2_CLK(cp0);
#ifdef B2INS_PHASE_CLOCKS
        if (!(p.debug & 1))
#endif
        {
          const int tj = base + j;
          const uint32_t t = t0 + static_cast<uint32_t>(tj);
          const bool live = tj < cnt;
          Normal2 z{0.0, 0.0};
          double m = 0.0;
          if (live) {
            z = normal_pair(t, c, mr.lo, mr.hi, p.k0, p.k1);
            m = (ref0[ref_off] + eb) + ew * z.z1;
            if (kSlow && any_vib)
              m += vib_term(e, ax, is_acc ? 0 : 1, t, mr.lo, mr.hi, p.k0, p.k1, mr.run, phase);
          }
          const double d = gm_block<kAvRound>(gb * z.z0, ga, apj, aG, j, carry);
          m += d + ewd * z.z0;
          int64_t row;
          if (kSlow && mr.warp_dumps && mr.dump && live && p.out_gyro && dump_row(p, t, &row))
            (is_acc ? p.out_accel : p.out_gyro)[mr.run * p.osr + row * p.ost + ax * p.osc] = m;
          out0[out_off] = m;
        }
        B2_CLK(cp1);
        B2_ACC(14, cp0, cp1);
        if (base + kAvRound >= cnt) {                      // last round of the tile: release the stage
          __syncwarp();
          if (lane == 0) mbar_arrive(&sm.empty[s]);
          ++tile;
          if (++s == kStagesFast) {
            s = 0;
            parity ^= 1u;
          }
          base = 0;
          t0 += kTile;
          ref_off = s * kTile * 3;
          cnt = static_cast<int>(min64(kTile, p.n - static_cast<int64_t>(t0)));
        } else {
          base += kAvRound;
          ref_off += kAvRound * 3;
        }
        out_off = (out_off == 2 * kSlotSet) ? 0 : out_off + kSlotSet;
        B2_CLK(cb0);
        stage_sync();                     // intervals 0 .. rounds end in a barrier
        B2_CLK(cb1);
        B2_ACC(15, cb0, cb1);
      }
      stage_sync();                       // interval `rounds`: A's last round; the one after is V's alone
    };
    if (mr.warp_dumps || any_vib)
      produce(std::true_type{});
    else
      produce(std::false_type{});
    return;
  }

  // initial state (both A and V derive what they need from it)
  const NavState st0 = mc_init<1>(p, mr.run);

  if (is_a) {
    // ================================= A: attitude =================================================
    AttState a;
    a.yaw = st0.yaw; a.pitch = st0.pitch; a.roll = st0.roll;
    a.sc = st0.sc;
    a.icp = st0.icp;
    if (mr.dump && j == 0 && p.out_att) put_att_row(p, mr.run, 0, a.yaw, a.pitch, a.roll);
    for (int64_t i = 0; i < rounds + 2; ++i) {
      B2_CLK(ca0);
#ifdef B2INS_PHASE_CLOCKS
      if (!(p.debug & 2))
#endif
      if (i >= 1 && i <= rounds) {
        const int64_t r0 = (i - 1) * kAvRound;
        const int sbuf = static_cast<int>((i - 1) % 3), rbuf = static_cast<int>((i - 1) & 1);
        // samples of this round that are followed by a step (the last sample of the series is not)
        const int kmax = static_cast<int>(min64(kAvRound, p.n - 1 - r0));
        auto ring_store = [&](int k) {                    // the sin/cos after step k, for V
          if (j == 0) {
            double* o = sm.ring[rbuf][k][grp];
            reinterpret_cast<double2*>(o)[0] = make_double2(a.sc.sy, a.sc.cy);
            reinterpret_cast<double2*>(o)[1] = make_double2(a.sc.sp, a.sc.cp);
            reinterpret_cast<double2*>(o)[2] = make_double2(a.sc.sr, a.sc.cr);
          }
        };
        auto a_step = [&](int k) {                        // one step with the exact path and the history rows
          const SampleSlot& sl = sm.slot[sbuf][k / G][lane - j + (k % G)];
          const Vec3 w{sl.g[0], sl.g[1], sl.g[2]};
          att_step(a, w, p.dt, ((r0 + k + 1) & (kResync - 1)) == 0);
          ring_store(k);
          int64_t row;
          if (mr.warp_dumps && mr.dump && j == 0 && p.out_att && dump_row(p, r0 + k + 1, &row))
            put_att_row(p, mr.run, row, wrap_once(a.yaw), a.pitch, wrap_once(a.roll));
        };
        if (mr.warp_dumps || kmax < kAvRound) {
#pragma unroll 1
          for (int k = 0; k < kmax; ++k) a_step(k);
        } else {
          // Blocks of four steps (spec_block).  The block's gyro samples are loaded at its start, so that no
          // shared load waits behind the ring stores of the step before.  A redone block rewrites the ring
          // with the same or the corrected values before V sees it (V reads after the next barrier).
#pragma unroll 1
          for (int kb = 0; kb < kAvRound; kb += kSpecBlock) {
            Vec3 w[kSpecBlock];
#pragma unroll
            for (int k = 0; k < kSpecBlock; ++k) {
              const SampleSlot& sl = sm.slot[sbuf][(kb + k) / G][lane - j + ((kb + k) % G)];
              w[k] = Vec3{sl.g[0], sl.g[1], sl.g[2]};
            }
            AttState saved;
            const bool redone = spec_block(true, a, saved, [&](int k) {
              const bool cold = att_step<true>(a, w[k], p.dt, false);
              ring_store(kb + k);
              return cold;
            }, [&](int k) { a_step(kb + k); });
            if (!redone && ((r0 + kb + kSpecBlock) & (kResync - 1)) == 0) {
              // the time-based re-evaluation (1 block of 16) falls on the block's last step: att_step's
              // exact path after it, as att_step(..., resync = true) takes it
              B2_CLK(cr0);
              att_exact(a);
              a.icp = rcp_nr(a.sc.cp) * p.dt;
              ring_store(kb + kSpecBlock - 1);
              B2_CLK(cr1);
              B2_ACC(10, cr0, cr1);
            }
          }
        }
      }
      B2_CLK(ca1);
      B2_ACC(8, ca0, ca1);
      if (i <= rounds) stage_sync();
      B2_CLK(ca2);
      B2_ACC(9, ca1, ca2);
    }
    if (mr.active && j == 0) put_end<true, false>(p, mr.run, a.yaw, a.pitch, a.roll, Vec3{}, Vec3{});
    return;
  }

  // =================================== V: velocity, position ========================================
  VelState v;
  v.vel_b = st0.vel_b;
  v.vel = st0.vel;
  v.pos = st0.pos;
  v.gdt = st0.g * p.dt;
  SinCos3 old = st0.sc;
  if (mr.dump && j == 0 && p.out_att) put_pv_row(p, mr.run, 0, v.pos, v.vel);
  for (int64_t i = 0; i < rounds + 2; ++i) {
    B2_CLK(cv0);
#ifdef B2INS_PHASE_CLOCKS
    if (!(p.debug & 4))
#endif
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
        if (hist && mr.dump && j == 0 && p.out_att && dump_row(p, r0 + k + 1, &row)) put_pv_row(p, mr.run, row, v.pos, v.vel);
      };
      if (mr.warp_dumps || kmax < kAvRound) {
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
    B2_CLK(cv1);
    B2_ACC(11, cv0, cv1);
    if (i <= rounds) stage_sync();        // V's last round follows the last barrier
    B2_CLK(cv2);
    B2_ACC(12, cv1, cv2);
  }
  if (mr.active && j == 0) put_end<false, true>(p, mr.run, 0.0, 0.0, 0.0, v.pos, v.vel);
}

}  // namespace b2ins
