// b2ins device-side common pieces: constants, Philox4x32-10 + Box-Muller (the
// "b2ins noise spec", DESIGN.md section 4), mbarrier / bulk-copy (TMA) PTX wrappers.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "fastmath64.cuh"

namespace b2ins {

// ---- WGS-84, geoparams.py:18-23 and :40-43 --------------------------------
constexpr double kRe = 6378137.0;
constexpr double kFlat = 1.0 / 298.257223563;
constexpr double kEcc = 0.0818191908426215;
constexpr double kESqr = kEcc * kEcc;
constexpr double kWie = 7292115e-11;
constexpr double kNormalGravity = 9.7803253359;
constexpr double kGravK = 0.00193185265241;
constexpr double kGravM = 0.00344978650684;
constexpr double kPi = 3.141592653589793238462643383279502884;
constexpr double kTwoPi = 2.0 * kPi;
constexpr double kHalfPi = 0.5 * kPi;

// ---- Philox4x32-10 ---------------------------------------------------------
// Counter words: (t, draw id, run_lo, run_hi); key = (seed_lo, seed_hi).
constexpr uint32_t kPhiloxM0 = 0xD2511F53u;
constexpr uint32_t kPhiloxM1 = 0xCD9E8D57u;
constexpr uint32_t kPhiloxW0 = 0x9E3779B9u;
constexpr uint32_t kPhiloxW1 = 0xBB67AE85u;

// draw ids (counter word 1); must match oracle/oracle_np.py
constexpr uint32_t kDrawAccel = 0;  // +axis: (GM drive, white)
constexpr uint32_t kDrawGyro = 3;   // +axis: (GM drive, white)
constexpr uint32_t kDrawVib = 6;    // +axis: (accel random vib, gyro random vib)
constexpr uint32_t kDrawPhase = 9;  // +axis, t = 0xFFFFFFFF: sinusoidal gyro-vib phase
constexpr uint32_t kDrawOdo = 12;   // odometer white noise (z0)
constexpr uint32_t kDrawMag = 13;   // magnetometer: 13 (x, y), 14 (z from z0)
constexpr uint32_t kDrawPsd = 16;   // +3*sensor+axis, t = bin index: PSD random phases
constexpr uint32_t kDrawRrw = 32;   // +3*sensor+axis: rate random walk drive (z0)
constexpr uint32_t kDrawQuant = 38; // +3*sensor+axis: quantisation uniform (words x1:x0, as uniform01)

struct PhiloxOut {
  uint32_t x0, x1, x2, x3;
};

__device__ __forceinline__ PhiloxOut philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2,
                                                   uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(kPhiloxM0, c0), lo0 = kPhiloxM0 * c0;
    const uint32_t hi1 = __umulhi(kPhiloxM1, c2), lo1 = kPhiloxM1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0;
    const uint32_t n2 = hi0 ^ c3 ^ k1;
    c0 = n0;
    c1 = lo1;
    c2 = n2;
    c3 = lo0;
    k0 += kPhiloxW0;
    k1 += kPhiloxW1;
  }
  return PhiloxOut{c0, c1, c2, c3};
}

// 52-bit uniforms built from the bit pattern (exact, no int->double conversion):
//   u_open0 = 1 - m*2^-52 in (0, 1]      u_half = m*2^-52 in [0, 1)
__device__ __forceinline__ double u01_from_bits(uint32_t lo, uint32_t hi) {
  // m = (hi:lo) >> 12
  const uint32_t mh = hi >> 12;
  const uint32_t ml = (hi << 20) | (lo >> 12);
  return __hiloint2double(0x3FF00000u | mh, ml) - 1.0;  // [0,1)
}
// v = 1 + m*2^-52 in [1, 2): u_half = v - 1 and u_open0 = 2 - v, both exact
__device__ __forceinline__ double one_plus_u01_from_bits(uint32_t lo, uint32_t hi) {
  const uint32_t mh = hi >> 12;
  const uint32_t ml = (hi << 20) | (lo >> 12);
  return __hiloint2double(0x3FF00000u | mh, ml);
}

struct Normal2 {
  double z0, z1;
};

// Box-Muller in float64 from one Philox output: r = sqrt(-2 ln u1), (z0, z1) = r (cos, sin)(2 pi u2),
// u1 = 1 - m1 2^-52 with m1 = (x1:x0) >> 12 and u2 = m2 2^-52 with m2 = (x3:x2) >> 12.
__device__ __forceinline__ Normal2 normal_from_words(const PhiloxOut& x) {
  const double u1 = 2.0 - one_plus_u01_from_bits(x.x0, x.x1);   // 1 - u in (0, 1], exact
  const double r = sqrt_nr(-2.0 * log_unit(u1));
  double s, c;
  sincospi_2u(fma(one_plus_u01_from_bits(x.x2, x.x3), 2.0, -2.0), &s, &c);    // 2 u2, u2 in [0, 1), exact
  return Normal2{r * c, r * s};
}

__device__ __forceinline__ Normal2 normal_pair(uint32_t t, uint32_t draw, uint32_t run_lo,
                                               uint32_t run_hi, uint32_t k0, uint32_t k1) {
  return normal_from_words(philox4x32_10(t, draw, run_lo, run_hi, k0, k1));
}

__device__ __forceinline__ double uniform01(uint32_t t, uint32_t draw, uint32_t run_lo,
                                            uint32_t run_hi, uint32_t k0, uint32_t k1) {
  const PhiloxOut x = philox4x32_10(t, draw, run_lo, run_hi, k0, k1);
  return u01_from_bits(x.x0, x.x1);
}

// ---- mbarrier + bulk async copy (TMA, 1-D) ---------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared bulk copy completing on an mbarrier; 16-byte aligned, bytes % 16 == 0
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// shared -> global bulk copy (bulk-group completion)
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem),
               "r"(smem_u32(src_smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_read0() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
__device__ __forceinline__ void bulk_wait0() {
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
__device__ __forceinline__ void fence_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__host__ __device__ __forceinline__ int64_t min64(int64_t a, int64_t b) { return a < b ? a : b; }

// ---- statistics with NumPy's non-finite rules (np.max, np.mean, np.std) ----
// max that keeps a NaN in either argument, as np.max does (fmax is IEEE maxNum: it drops the NaN)
__device__ __forceinline__ double max_nan(double a, double b) { return (a > b || a != a) ? a : b; }
// a running mean m moved toward the sample or partial mean x by the step d * f (d = x - m); when d is not
// finite (x or m is +-inf or NaN) the mean is m + x instead: +-inf for infinities of one sign, NaN for a NaN
// or for both signs, as np.mean of the samples (the finite step would make inf - inf = NaN of a lone inf)
__device__ __forceinline__ double mean_step(double m, double x, double d, double f) {
  return isfinite(d) ? fma(d, f, m) : m + x;
}

// 64-bit shuffle within a lane group of width W
template <int W>
__device__ __forceinline__ double shfl_grp(double v, int src) {
  return __shfl_sync(0xffffffffu, v, src, W);
}

// ---- block-wide affine scan of a Gauss-Markov recurrence, C channels, W warps ----
// Thread i holds the map x -> sA x + sE of its stretch of samples; the stretches compose in thread order
// by (A, E) o (A', E') = (A A', A' E + E').  Two halves around the caller's __syncthreads:
// warp half: the inclusive scan within the warp, and lane 31 leaves the warp's total in wtot[C][W][2].
template <int C, int W>
__device__ __forceinline__ void affine_scan_warp(double (&sA)[C], double (&sE)[C], double (*wtot)[W][2], int lane,
                                                 int warp) {
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const double uA = __shfl_up_sync(0xffffffffu, sA[c], off);
      const double uE = __shfl_up_sync(0xffffffffu, sE[c], off);
      if (lane >= off) {
        sE[c] = fma(sA[c], uE, sE[c]);
        sA[c] *= uA;
      }
    }
  }
  if (lane == 31) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      wtot[c][warp][0] = sA[c];
      wtot[c][warp][1] = sE[c];
    }
  }
}

// block half, after the barrier: S = the state at this thread's first sample (the warps before it, then the
// lanes before it, applied to carry, the state at the block's first sample), and carry advanced over the whole
// block -- by every thread alike, so every thread holds the same next carry
template <int C, int W>
__device__ __forceinline__ void affine_scan_block(const double (&sA)[C], const double (&sE)[C],
                                                  const double (*wtot)[W][2], int lane, int warp, double (&carry)[C],
                                                  double (&S)[C]) {
#pragma unroll
  for (int c = 0; c < C; ++c) {
    double pA = 1.0, pE = 0.0;
    for (int w = 0; w < warp; ++w) {
      pE = fma(wtot[c][w][0], pE, wtot[c][w][1]);
      pA *= wtot[c][w][0];
    }
    const double lA = __shfl_up_sync(0xffffffffu, sA[c], 1), lE = __shfl_up_sync(0xffffffffu, sE[c], 1);
    if (lane > 0) {
      pE = fma(lA, pE, lE);
      pA *= lA;
    }
    S[c] = fma(pA, carry[c], pE);
    double tA = 1.0, tE = 0.0;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      tE = fma(wtot[c][w][0], tE, wtot[c][w][1]);
      tA *= wtot[c][w][0];
    }
    carry[c] = fma(tA, carry[c], tE);
  }
}

}  // namespace b2ins
