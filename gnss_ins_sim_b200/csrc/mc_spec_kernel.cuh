// K12, warp-specialised form: sample PRODUCER warps and INTEGRATOR warps on different SM
// sub-partitions.
//
// The Monte-Carlo step has a time-parallel part (Philox + Box-Muller normals, Gauss-Markov scan:
// ~440 FP64 instructions per sample, no dependency between samples) and a serial part (the
// strapdown recurrence: ~90 FP64 instructions per step on a ~100-cycle dependency chain).  One warp
// doing both leaves its scheduler's FP64 pipe idle during the chain and the chain idle during the
// noise.  Here a CTA is WI integrator warps plus P producer warps per integrator warp:
//
//   * an integrator warp owns 32/G runs (G lanes per run, state replicated across the group as in
//     mc_kernel) and does nothing but steps, reading complete measurements from shared-memory slots;
//   * its P producers own 6/P of the six channels (accel xyz, gyro xyz) each: Philox, Box-Muller,
//     white noise, bias, vibration, the Gauss-Markov drift of THEIR channels (the scan state lives in
//     the producer), for the same 32 (run, sample) lanes, one pass of G samples at a time, and own the
//     TMA tile pipeline of the shared true trajectory;
//   * with CTAs of four warps (WI (1 + P) = 4) every warp has an SM sub-partition -- its FP64 pipe,
//     its issue slots -- to itself, and nothing but the slot hand-over couples them: a named barrier
//     of 32 (1 + P) threads per round of kRound samples, slots double-buffered so that the producers
//     fill round r + 1 while round r is integrated.
//
// Which (G, P, WI) is used for how many runs is measured, not guessed: b2ins_api.cu, auto_lanes() and
// default_shape() (ref_frame 1 with groups of 4 and 8 lanes takes mc_av_kernel.cuh instead).
#pragma once
#include "mc_kernel.cuh"

namespace b2ins {

template <int G, int P, int WI>
struct SpecShape {
  static constexpr int kRound = (G >= 8) ? G : 8;     // samples per run handed over at a time
  static constexpr int kPasses = kRound / G;          // passes of G samples per round
  // P = 6, WI = 1: warps 1..3 and 5..7 produce, warp 4 (which would share the integrator's SM
  // sub-partition) has nothing to do and leaves at once
  static constexpr bool kSpare = (P == 6 && WI == 1);
  static constexpr int kThreads = (WI * (1 + P) + (kSpare ? 1 : 0)) * 32;
  static constexpr int kChan = 6 / P;                 // channels per producer warp
  // speculative blocks (spec_block, mech.cuh): groups of 4 and 8 lanes, the shapes of the few-runs
  // configurations, which run without a register cap
  static constexpr bool kSpec = (G == 4 || G == 8);
  static_assert(6 % P == 0 && kTile % kRound == 0 && 32 % G == 0, "shape");
};

template <int G, int P, int WI>
struct SpecSmem {
  alignas(128) double gyro[kStagesFast][kTile * 3];
  alignas(128) double accel[kStagesFast][kTile * 3];
  alignas(16) SampleSlot slot[2][SpecShape<G, P, WI>::kPasses][WI][32];
  // the state before a speculative block (integrator lanes; one dummy element where there are none)
  alignas(16) NavState saved[SpecShape<G, P, WI>::kSpec ? WI : 1][SpecShape<G, P, WI>::kSpec ? 32 : 1];
  alignas(8) uint64_t full[kStagesFast];
  alignas(8) uint64_t empty[kStagesFast];
};

template <int G, int RF, int P, int WI, bool SPLIT, int MINB>
__global__ void __launch_bounds__(SpecShape<G, P, WI>::kThreads, MINB)
mc_spec_kernel(const __grid_constant__ McParams p) {
  using Sh = SpecShape<G, P, WI>;
  static_assert(!SPLIT || G >= 4, "lane roles need groups of four");
  __shared__ SpecSmem<G, P, WI> sm;
  constexpr int kRunsPerWarp = 32 / G;
  constexpr int kChan = Sh::kChan;
  const int lane = threadIdx.x & 31;
  const int pwarp = threadIdx.x >> 5;
  const bool integrator = pwarp < WI;
  // producer number 0 .. WI P - 1 (the spare warp 4 of the P = 6 shape is skipped)
  const int pidx = Sh::kSpare ? (pwarp < 4 ? pwarp - 1 : pwarp - 2) : pwarp - WI;
  const int gi = integrator ? pwarp : pidx / P;            // the integrator warp this warp works for
  const int pp = integrator ? 0 : pidx % P;                // producer index within the group
  const int j = lane % G;
  const int role = lane & 3;
  const McRun mr = mc_run(p, (static_cast<int64_t>(blockIdx.x) * WI + gi) * kRunsPerWarp + lane / G);
  // (the odometer variant, cfg.algo = 1, takes the single-warp form: mc_kernel)
  const int64_t num_tiles = (p.n + kTile - 1) / kTile;
  const int issuer = WI * 32;                              // lane 0 of the first producer warp
  auto group_sync = [&]() { asm volatile("bar.sync %0, %1;" ::"r"(1 + gi), "n"(32 * (1 + P)) : "memory"); };

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStagesFast; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], WI * P);
    }
    mbar_fence_init();
  }
  __syncthreads();
  if (Sh::kSpare && pwarp == 4) return;

  if (!integrator) {
    // =============================== producer ===============================================
    if (threadIdx.x == issuer)
      for (int s = 0; s < kStagesFast && s < num_tiles; ++s) issue_tile<false, false>(sm, p, s, s);
    // error model of this producer's channels (c < 3: accel axis c, else gyro axis c - 3)
    double carry[kChan], apj[kChan], aG[kChan];
#pragma unroll
    for (int q = 0; q < kChan; ++q) {
      const int c = pp * kChan + q;
      const double a = (c < 3) ? p.accel.gm_a[c % 3] : p.gyro.gm_a[c % 3];
      carry[q] = 0.0;                                   // d[0] = 0
      apj[q] = (G > 1) ? ipow(a, j) : 1.0;
      aG[q] = (G > 1) ? ipow(a, G) : a;
    }
    double phase[3] = {0.0, 0.0, 0.0};
    if (p.gyro.vib_type == 2) {
#pragma unroll
      for (int c = 0; c < 3; ++c)  // np.random.rand(1)*2*pi, pathgen.py:553-555
        phase[c] = (uniform01(0xFFFFFFFFu, kDrawPhase + c, mr.lo, mr.hi, p.k0, p.k1) * 2.0) * kPi;
    }
    const bool any_vib = (p.accel.vib_type | p.gyro.vib_type) != 0;
    int rnd = 0;
    for (int64_t tile = 0; tile < num_tiles; ++tile) {
      const int s = static_cast<int>(tile % kStagesFast);
      const uint32_t parity = static_cast<uint32_t>((tile / kStagesFast) & 1);
      const int64_t t0 = tile * kTile;
      const int cnt = static_cast<int>(min64(kTile, p.n - t0));
      refill_and_wait<false, false>(sm, p, threadIdx.x == issuer, static_cast<int>(tile),
                                    static_cast<int>(num_tiles), s, parity, 0);
      for (int base = 0; base < cnt; base += Sh::kRound, ++rnd) {
        const int buf = rnd & 1;
        B2_CLK(cp0);
#ifdef B2INS_PHASE_CLOCKS
        if (p.debug & 1) { group_sync(); continue; }   // isolate the integrator
#endif
        // two passes at a time, the Box-Muller pairs of both (and of all channels) first --
        // unconditionally: a sample past the end costs nothing and is dropped --: independent chains
        // the scheduler interleaves
        constexpr int kIlp = (G >= 4 && Sh::kPasses >= 2) ? 2 : 1;     // (narrow groups run under a register cap)
#pragma unroll 1
        for (int b0 = 0; b0 < Sh::kPasses; b0 += kIlp) {
          Normal2 z[kIlp][kChan];
#pragma unroll
          for (int bi = 0; bi < kIlp; ++bi)
#pragma unroll
            for (int q = 0; q < kChan; ++q) {
              z[bi][q] = Normal2{0.0, 0.0};
              if (kIlp > 1 || base + (b0 + bi) * G + j < cnt)
                z[bi][q] = normal_pair(static_cast<uint32_t>(t0 + base + (b0 + bi) * G + j), pp * kChan + q, mr.lo,
                                       mr.hi, p.k0, p.k1);
            }
#pragma unroll
          for (int bi = 0; bi < kIlp; ++bi) {
            const int b = b0 + bi;
            const int tj = base + b * G + j;
            const int64_t t = t0 + tj;
            const bool live = tj < cnt;
            SampleSlot& mine = sm.slot[buf][b][gi][lane];
#pragma unroll
            for (int q = 0; q < kChan; ++q) {
              const int c = pp * kChan + q;
              const int ax = c % 3;
              const bool is_acc = c < 3;
              const TriadNoise& e = is_acc ? p.accel : p.gyro;
              const double z0 = (kIlp > 1 && !live) ? 0.0 : z[bi][q].z0;
              double m = 0.0;
              if (live) {
                const double ref = is_acc ? sm.accel[s][tj * 3 + ax] : sm.gyro[s][tj * 3 + ax];
                m = (ref + e.b[ax]) + e.w[ax] * z[bi][q].z1;
                if (any_vib)
                  m += vib_term(e, ax, is_acc ? 0 : 1, static_cast<uint32_t>(t), mr.lo, mr.hi, p.k0, p.k1,
                                mr.run, phase);
              }
              // + drift: the GM state d[t] (pathgen.py:583-590) or drift*z[t] if tau = inf (:591-593)
              const double d = gm_block<G>(e.gm_b[ax] * z0, e.gm_a[ax], apj[q], aG[q], j, carry[q]);
              m += d + e.wd[ax] * z0;
              int64_t row;
              if (mr.warp_dumps && mr.dump && live && p.out_gyro && dump_row(p, t, &row))
                (is_acc ? p.out_accel : p.out_gyro)[mr.run * p.osr + row * p.ost + ax * p.osc] = m;
              if (is_acc) mine.a[ax] = m; else mine.g[ax] = m;
            }
          }
        }
        B2_CLK(cp1);
        B2_ACC(7, cp0, cp1);
        group_sync();   // round rnd is complete; the integrator has finished round rnd - 1
        B2_CLK(cp2);
        B2_ACC(6, cp1, cp2);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.empty[s]);
    }
    return;
  }

  // ================================= integrator ===============================================
  NavState st = mc_init<RF>(p, mr.run);
  if (mr.dump && j == 0 && p.out_att) put_state_row(p, mr.run, 0, st.yaw, st.pitch, st.roll, st.pos, st.vel);
  int rnd = 0;
  for (int64_t tile = 0; tile < num_tiles; ++tile) {
    const int64_t t0 = tile * kTile;
    const int cnt = static_cast<int>(min64(kTile, p.n - t0));
    for (int base = 0; base < cnt; base += Sh::kRound, ++rnd) {
      B2_CLK(ci0);
      group_sync();   // the samples of round rnd are in slot set rnd & 1
      B2_CLK(ci1);
      B2_ACC(4, ci0, ci1);
      const int buf = rnd & 1;
#ifdef B2INS_PHASE_CLOCKS
      if (p.debug & 2) continue;                       // isolate the producers
#endif
#pragma unroll 1
      for (int b = 0; b < Sh::kPasses; ++b) {
        const int pb = base + b * G;
        if (pb >= cnt) break;
        // samples of this pass that are followed by a step (the last sample of the series is not)
        const int kmax = static_cast<int>(min64(min64(G, cnt - pb), p.n - 1 - (t0 + pb)));
        const SampleSlot* grp = &sm.slot[buf][b][gi][lane - j];
        double keep[9];  // lane k keeps the state after sample pb + k (history output)
#pragma unroll
        for (int c = 0; c < 9; ++c) keep[c] = 0.0;
        auto one_step = [&](int k, bool hist) {
          const SampleSlot& sl = grp[k];
          const Vec3 w{sl.g[0], sl.g[1], sl.g[2]};
          const Vec3 f{sl.a[0], sl.a[1], sl.a[2]};
          const bool resync = ((t0 + pb + k + 1) & (kResync - 1)) == 0;
          nav_step<RF, SPLIT, 0>(st, w, f, p.dt, p.earth_rot != 0, role, resync);
          if (hist && j == k) keep_state(keep, st);
        };
        if (mr.warp_dumps) {         // history output: the rare path keeps the simple loop
#pragma unroll 1
          for (int k = 0; k < kmax; ++k) one_step(k, true);
          const int tj = pb + j;
          if (mr.dump && tj < cnt) put_kept_row(p, mr.run, t0 + tj, keep);
        } else if (G == 1) {
          if (kmax > 0) one_step(0, false);
        } else if (Sh::kSpec && kmax == G) {
          // blocks of four steps, speculated unless the block holds a time-based re-evaluation (1 of 16)
#pragma unroll 1
          for (int kb = 0; kb < G; kb += kSpecBlock) {
            const bool speculate = ((t0 + pb + kb) & (kResync - 1)) + kSpecBlock < kResync;
            spec_block(speculate, st, sm.saved[gi][lane], [&](int k) {
              const SampleSlot& sl = grp[kb + k];
              const Vec3 w{sl.g[0], sl.g[1], sl.g[2]};
              const Vec3 f{sl.a[0], sl.a[1], sl.a[2]};
              return nav_step<RF, SPLIT, 0, true>(st, w, f, p.dt, p.earth_rot != 0, role, false);
            }, [&](int k) { one_step(kb + k, false); });
          }
        } else {
          // two steps per iteration: the off-chain tail of step k overlaps the chain of step k + 1
          int k = 0;
#pragma unroll 1
          for (; k + 1 < kmax; k += 2) {
            one_step(k, false);
            one_step(k + 1, false);
          }
          if (k < kmax) one_step(k, false);
        }
      }
      B2_CLK(ci2);
      B2_ACC(5, ci1, ci2);
    }
  }

  // ---- per-run results ---------------------------------------------------------------------
  if (mr.active && j == 0) {
    put_end<true, true>(p, mr.run, st.yaw, st.pitch, st.roll, st.pos, st.vel);
  }
}

}  // namespace b2ins
