// K8: magnetometer measurement generator.  Replaces pathgen.mag_gen (gnss_ins_sim/pathgen/pathgen.py:643-661)
// for all Monte-Carlo runs at once: mag[r][k] = si (ref_mag[k] + hi) + std * N(0,1).
// Noise spec: the Box-Muller pair (k, 13, global run) gives (z_x, z_y); the pair (k, 14, global run)
// gives z_z from its z0 (its z1 is unused).  One thread per (run, sample), the sample index fastest so
// that the 24 B stores of a warp are contiguous; ref_mag [n][3] is shared by every run (L2-resident).
// Two Philox + Box-Muller pairs per 24 B written: DESIGN.md section 3 says which bound it sits at.
#pragma once
#include "common.cuh"

namespace b2ins {

struct MagParams {
  int64_t n, runs, run_offset;
  const double* ref;   // [n][3]
  double* out;         // [runs][n][3]
  double si[9];        // row-major
  double hi[3], std[3];
  uint32_t k0, k1;
};

// Sample k of global run (rl, rh): si (ref_mag[k] + hi) + std * z.  K8 writes it and K10 (magcal_kernel.cuh)
// regenerates it, so a calibration of generated runs sees exactly the samples get_data(['mag']) returns.
__device__ __forceinline__ void mag_sample(const double* ref_mag, const double* si, const double* hi,
                                           const double* std, int64_t k, uint32_t rl, uint32_t rh, uint32_t k0,
                                           uint32_t k1, double o[3]) {
  const Normal2 zxy = normal_pair(static_cast<uint32_t>(k), kDrawMag, rl, rh, k0, k1);
  const Normal2 zz = normal_pair(static_cast<uint32_t>(k), kDrawMag + 1, rl, rh, k0, k1);
  const double* ref = ref_mag + k * 3;
  const double m0 = ref[0] + hi[0], m1 = ref[1] + hi[1], m2 = ref[2] + hi[2];
  o[0] = (si[0] * m0 + si[1] * m1 + si[2] * m2) + std[0] * zxy.z0;
  o[1] = (si[3] * m0 + si[4] * m1 + si[5] * m2) + std[1] * zxy.z1;
  o[2] = (si[6] * m0 + si[7] * m1 + si[8] * m2) + std[2] * zz.z0;
}

__global__ void __launch_bounds__(256) mag_noise_kernel(const __grid_constant__ MagParams p) {
  const int64_t total = p.n * p.runs;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / p.n;
    const int64_t k = i - r * p.n;
    const uint64_t run = static_cast<uint64_t>(p.run_offset + r);
    double o[3];
    mag_sample(p.ref, p.si, p.hi, p.std, k, static_cast<uint32_t>(run), static_cast<uint32_t>(run >> 32), p.k0,
               p.k1, o);
    double* out = p.out + i * 3;
    out[0] = o[0];
    out[1] = o[1];
    out[2] = o[2];
  }
}

}  // namespace b2ins
