// K1: IMU sensor-error generator, materialised -- pathgen.acc_gen / gyro_gen / bias_drift
// (pathgen.py:441-594).  One CTA per (run, time segment) walks the samples in tiles of kNoiseTile;
// thread i makes the kNoisePer consecutive samples i kNoisePer .. of the tile, one after the other:
// six Box-Muller pairs per sample (Philox4x32-10), the measurement without the drift at the start of
// its stretch staged in shared memory, the Gauss-Markov recurrence d[t+1] = a d[t] + b z[t] run
// serially inside the stretch (one FMA per sample and channel).  What the stretches owe each other is
// an affine scan over the 128 threads of a tile -- shuffles within a warp, four warp totals through
// shared memory: ONE exchange per kNoisePer samples instead of one per sample -- after which every
// thread adds a^q S to its samples and the tile leaves shared memory in the caller's layout with
// coalesced stores.  imu_err_stats_kernel (K9, sensor_stats_kernel.cuh) reduces the tile instead of
// storing it; it calls noise_prologue and the scan of common.cuh, and repeats only the stretch loop
// (triad_sample into the stage): with that loop in a shared function the compiler allocates K9's
// registers differently, so a change to the loop here goes there too.
#pragma once
#include "mc_kernel.cuh"

namespace b2ins {

constexpr int kNoiseThreads = 128;
constexpr int kNoiseWarps = kNoiseThreads / 32;
constexpr int kNoisePer = 7;                               // consecutive samples per thread and tile
constexpr int kNoiseTile = kNoiseThreads * kNoisePer;      // 896 samples per tile (the staged tile fits 48 KB)

struct NoiseParams {
  int64_t n, runs, run_offset;
  double dt;
  uint32_t k0, k1;
  TriadNoise gyro, accel;
  const double* ref_gyro;
  const double* ref_accel;
  double* out_gyro;
  double* out_accel;
  int64_t osr, ost, osc;
  double* z_dump;  // [runs][n][12] or null
  // time segmentation (few runs, long series): blockIdx.x = run * nseg + seg, samples
  // [seg*seg_len, min(n, (seg+1)*seg_len)).  pass 0: write outputs, GM state at the segment
  // start taken from seg_carry[run][seg][6] (all zero for seg 0); pass 1: no output, only the
  // zero-state GM response at the segment end -> seg_end[run][seg][6].  Pass 1 covers segments
  // 0 .. nseg-2 only (the end value of the last one is never used: blockIdx.x = run * (nseg-1) +
  // seg) and only their last pass1_len samples: older drives have decayed below 1e-20 of the
  // state (pass1_len = seg_len if the correlation time is too long for that)
  int64_t seg_len;
  int64_t pass1_len;
  int nseg;
  int pass;
  double* seg_carry;
  double* seg_end;
};

// one triad (three channels of one sensor) of one sample: the measurement without the drift at the start of
// the thread's stretch, and the stretch's zero-state drift response advanced by one sample
template <int SENSOR>   // 0 accel (draws 0..2), 1 gyro (draws 3..5)
__device__ __forceinline__ void triad_sample(const NoiseParams& p, const TriadNoise& e, const double* ref3, uint32_t t,
                                             uint32_t run_lo, uint32_t run_hi, int64_t run, const double* phase,
                                             bool drives_only, double* r3, double* out3) {
  Normal2 z[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) z[c] = normal_pair(t, 3 * SENSOR + c, run_lo, run_hi, p.k0, p.k1);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double m = 0.0;
    if (!drives_only) {
      m = (ref3[c] + e.b[c]) + e.w[c] * z[c].z1;
      if (p.accel.vib_type | p.gyro.vib_type)   // uniform branch, off in the BASELINE configs
        m += vib_term(e, c, SENSOR, t, run_lo, run_hi, p.k0, p.k1, run, phase);
    }
    out3[c] = m + r3[c] + e.wd[c] * z[c].z0;        // + zero-state drift of the stretch (+ white drift)
    r3[c] = fma(e.gm_a[c], r3[c], e.gm_b[c] * z[c].z0);
  }
}

// the prologue of a K1 or K9 CTA, before its first __syncthreads: a^q per channel into apow[kNoisePer + 1][6],
// the run's sinusoidal gyro-vibration phase and, with carry_in, the Gauss-Markov state at the segment start
// (zero without)
__device__ __forceinline__ void noise_prologue(const NoiseParams& p, double (*apow)[6], int64_t run, int seg,
                                               uint32_t run_lo, uint32_t run_hi, bool carry_in, double (&phase)[3],
                                               double (&carry)[6]) {
  const int tid = threadIdx.x;
  if (tid < 6) {
    const double a = (tid < 3) ? p.accel.gm_a[tid] : p.gyro.gm_a[tid - 3];
    double v = 1.0;
    for (int q = 0; q <= kNoisePer; ++q) {
      apow[q][tid] = v;
      v *= a;
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) phase[c] = 0.0;
  if (p.gyro.vib_type == 2) {
#pragma unroll
    for (int c = 0; c < 3; ++c)
      phase[c] = (uniform01(0xFFFFFFFFu, kDrawPhase + c, run_lo, run_hi, p.k0, p.k1) * 2.0) * kPi;
  }
#pragma unroll
  for (int c = 0; c < 6; ++c) carry[c] = 0.0;
  if (carry_in && p.seg_carry) {
#pragma unroll
    for (int c = 0; c < 6; ++c) carry[c] = p.seg_carry[(run * p.nseg + seg) * 6 + c];
  }
}

__global__ void __launch_bounds__(kNoiseThreads, 4) imu_noise_kernel(const __grid_constant__ NoiseParams p) {
  __shared__ double stage[2][kNoiseTile * 3];     // accel, gyro of the tile, [sample][axis]
  __shared__ double wtot[6][kNoiseWarps][2];      // (A, E) of every warp's stretch, per channel
  __shared__ double apow[kNoisePer + 1][6];       // a^q per channel
  const int segs = (p.pass == 1) ? p.nseg - 1 : p.nseg;
  const int64_t run = blockIdx.x / segs;
  const int seg = static_cast<int>(blockIdx.x % segs);
  const int64_t seg_hi = min64(p.n, (seg + 1) * p.seg_len);
  const int64_t seg_lo = (p.pass == 1) ? seg_hi - p.pass1_len : seg * p.seg_len;
  const int64_t grun = p.run_offset + run;
  const uint32_t run_lo = static_cast<uint32_t>(grun), run_hi = static_cast<uint32_t>(grun >> 32);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double phase[3], carry[6];                      // carry: d at the first sample of the tile
  noise_prologue(p, apow, run, seg, run_lo, run_hi, p.pass == 0, phase, carry);
  __syncthreads();

  for (int64_t tile0 = seg_lo; tile0 < seg_hi; tile0 += kNoiseTile) {
    const int cnt = static_cast<int>(min64(kNoiseTile, seg_hi - tile0));
    // ---- the thread's stretch: one sensor triad at a time (three Box-Muller chains in flight) -------
    double r[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    int mine = cnt - tid * kNoisePer;                 // live samples of this thread's stretch
    mine = mine < 0 ? 0 : (mine > kNoisePer ? kNoisePer : mine);
#pragma unroll 1
    for (int q = 0; q < mine; ++q) {
      const int el = tid * kNoisePer + q;
      const int64_t t = tile0 + el;
      double m3[3];
      triad_sample<0>(p, p.accel, p.ref_accel + t * 3, static_cast<uint32_t>(t), run_lo, run_hi, run, phase,
                      p.pass == 1, r, m3);
#pragma unroll
      for (int c = 0; c < 3; ++c) stage[0][el * 3 + c] = m3[c];
      triad_sample<1>(p, p.gyro, p.ref_gyro + t * 3, static_cast<uint32_t>(t), run_lo, run_hi, run, phase,
                      p.pass == 1, r + 3, m3);
#pragma unroll
      for (int c = 0; c < 3; ++c) stage[1][el * 3 + c] = m3[c];
    }
    // ---- affine scan over the threads, six channels: (A, E) o (A', E') = (A A', A' E + E') -------
    double sA[6], sE[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      sA[c] = apow[mine][c];
      sE[c] = r[c];
    }
    affine_scan_warp<6, kNoiseWarps>(sA, sE, wtot, lane, warp);
    __syncthreads();   // warp totals; the staged tile is complete
    double S[6];       // drift at the first sample of this thread's stretch
    affine_scan_block<6, kNoiseWarps>(sA, sE, wtot, lane, warp, carry, S);
    if (p.pass == 0) {
      // ---- + a^q S on the thread's own samples, then the tile leaves in the caller's layout -------
#pragma unroll 1
      for (int q = 0; q < mine; ++q) {
        const int el = tid * kNoisePer + q;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          stage[0][el * 3 + c] += apow[q][c] * S[c];
          stage[1][el * 3 + c] += apow[q][3 + c] * S[3 + c];
        }
      }
      __syncthreads();
      const int64_t base = run * p.osr + tile0 * p.ost;
      if (p.osc == 1 && p.ost == 3) {            // [R][n][3]: the staged tile is the output, verbatim
        for (int e = tid; e < cnt * 3; e += kNoiseThreads) {
          p.out_accel[base + e] = stage[0][e];
          p.out_gyro[base + e] = stage[1][e];
        }
      } else {                                   // channel-major / time-major: consecutive threads, consecutive t
#pragma unroll
        for (int c = 0; c < 3; ++c)
          for (int el = tid; el < cnt; el += kNoiseThreads) {
            p.out_accel[base + el * p.ost + c * p.osc] = stage[0][el * 3 + c];
            p.out_gyro[base + el * p.ost + c * p.osc] = stage[1][el * 3 + c];
          }
      }
      if (p.z_dump) {
        // (acc_gm[3], acc_w[3], gyr_gm[3], gyr_w[3]) of every sample, recovered from the same Philox draws
        for (int el = tid; el < cnt; el += kNoiseThreads) {
          const int64_t t = tile0 + el;
          double* zd = p.z_dump + (run * p.n + t) * 12;
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const Normal2 za = normal_pair(static_cast<uint32_t>(t), kDrawAccel + c, run_lo, run_hi, p.k0, p.k1);
            const Normal2 zg = normal_pair(static_cast<uint32_t>(t), kDrawGyro + c, run_lo, run_hi, p.k0, p.k1);
            zd[c] = za.z0;
            zd[3 + c] = za.z1;
            zd[6 + c] = zg.z0;
            zd[9 + c] = zg.z1;
          }
        }
      }
    }
    __syncthreads();   // the stage and the warp totals are rewritten by the next tile
  }
  if (p.pass == 1 && threadIdx.x == 0) {
    // the tiles of a segment are whole (seg_len is a multiple of the tile) except in the last
    // segment, whose end value is never used
#pragma unroll
    for (int c = 0; c < 6; ++c) p.seg_end[(run * p.nseg + seg) * 6 + c] = carry[c];
  }
}

// carry-in of every segment from the zero-state segment responses: c[s+1] = a^L c[s] + E[s]
__global__ void noise_carry_kernel(NoiseParams p) {
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= p.runs * 6) return;
  const int64_t run = idx / 6;
  const int c = static_cast<int>(idx % 6);
  const double a = (c < 3) ? p.accel.gm_a[c] : p.gyro.gm_a[c - 3];
  const double aL = pow(a, static_cast<double>(p.seg_len));
  double cin = 0.0;
  for (int s = 0; s < p.nseg; ++s) {
    p.seg_carry[(run * p.nseg + s) * 6 + c] = cin;
    if (s + 1 < p.nseg) cin = aL * cin + p.seg_end[(run * p.nseg + s) * 6 + c];
  }
}

}  // namespace b2ins
