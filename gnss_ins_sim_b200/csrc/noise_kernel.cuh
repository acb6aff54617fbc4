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
// storing it: both bodies make their CTA's prologue with noise_prologue and every tile up to the end of
// the scan with noise_tile, and differ only in what they do with the finished tile.
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

// The IEEE Std 952 terms of b2ins_noise_terms, digested per channel in K1's order (accel x y z, gyro x y z)
struct NoiseTerms {
  double q[6];          // Q sqrt(12): the angle / velocity quantisation error is q (u - 1/2)
  double k[6];          // K sqrt(dt): the rate random walk's step per unit normal
  double r[6];          // R: the rate ramp R (t dt)
  double* seg_carry;    // time segments: the walk at every segment start [runs][nseg][6] (all zero for seg 0)
  double* seg_end;      //                pass 1: the zero-state walk at every segment end [runs][nseg][6]
};

// the terms of one triad of sample t, added to the measurement m3: the stretch's zero-state walk rk (then
// advanced by one sample), the quantisation rate error (e[t+1] - e[t]) / dt (qe: e[t], then e[t+1]) and the ramp.
// drives_only (pass 1): only the walk advances.  A channel whose k (q) is zero makes no walk (quantisation) draw:
// the branches are uniform over the launch, so a ramp alone costs no Philox.
template <int SENSOR>
__device__ __forceinline__ void terms_sample(const NoiseParams& p, const NoiseTerms& x, int64_t t, uint32_t run_lo,
                                             uint32_t run_hi, bool drives_only, double* rk, double* qe, double* m3) {
  const uint32_t t32 = static_cast<uint32_t>(t);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int ch = 3 * SENSOR + c;
    if (!drives_only) {
      double qr = 0.0;
      if (x.q[ch] != 0.0) {
        const double e1 = x.q[ch] * (uniform01(t32 + 1u, kDrawQuant + ch, run_lo, run_hi, p.k0, p.k1) - 0.5);
        qr = (e1 - qe[c]) / p.dt;
        qe[c] = e1;
      }
      m3[c] += rk[c] + (qr + x.r[ch] * (static_cast<double>(t) * p.dt));
    }
    if (x.k[ch] != 0.0) rk[c] = fma(x.k[ch], normal_pair(t32, kDrawRrw + ch, run_lo, run_hi, p.k0, p.k1).z0, rk[c]);
  }
}

// The run-to-run errors of b2ins_run_err (DESIGN.md section 4): the 1-sigma values of one sensor, SI units
struct RunErrSigma {
  double b[3];          // turn-on bias
  double sf[3];         // scale factor
  double ma[3][3];      // misalignment: sensitivity of sensor axis i to true axis j (zero diagonal)
};
struct RunErrs {
  RunErrSigma s[2];     // accel, gyro
};

// pair j (0..5) of one sensor's run errors, drawn from the global run id: e12 = (S row-major [9], b_run [3]) with
// S = diag(sf) + ma.  j < 3: (z0, z1) -> (b_run[j], sf[j]); j >= 3: the off-diagonals of row j - 3 in column order.
// K1's and K9's prologues (one thread per pair) and imu_run_err_kernel (one thread per sensor) share it.
__device__ __forceinline__ void run_err_pair(const RunErrSigma& s, int sensor, int j, uint32_t run_lo,
                                             uint32_t run_hi, uint32_t k0, uint32_t k1, double* e12) {
  const Normal2 z = run_err_normals(sensor, j, run_lo, run_hi, k0, k1);
  if (j < 3) {
    e12[9 + j] = s.b[j] * z.z0;
    e12[4 * j] = s.sf[j] * z.z1;
  } else {
    const int i = j - 3, c0 = (i == 0) ? 1 : 0, c1 = (i == 2) ? 1 : 2;
    e12[3 * i + c0] = s.ma[i][c0] * z.z0;
    e12[3 * i + c1] = s.ma[i][c1] * z.z1;
  }
}

// + delta[c] = b_run[c] + sum_j S[c][j] ref[j] on one triad; e12 in shared memory (broadcast reads)
__device__ __forceinline__ void run_err_add(const double* e12, const double* ref3, double* m3) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double d = e12[9 + c];
#pragma unroll
    for (int j = 0; j < 3; ++j) d = fma(e12[3 * c + j], ref3[j], d);
    m3[c] += d;
  }
}

// what a K1 or K9 CTA works on: its run, its time segment and that segment's samples [seg_lo, seg_hi), and the
// halves of the global run id that key its draws
struct NoiseCta {
  int64_t run, seg_lo, seg_hi;
  int seg;
  uint32_t run_lo, run_hi;
};

// The prologue of a K1 or K9 CTA, up to and including its first __syncthreads.  blockIdx.x = run * segs + seg:
// segs = nseg, or nseg - 1 in K1's pass 1, which covers only the last pass1_len samples of a segment (K9 runs
// pass 0 only).  It writes a^q per channel into apow[kNoisePer + 1][6], the run's sinusoidal gyro-vibration
// phase, and carry: the Gauss-Markov state (and under TERMS the walk) at the segment start, zero in pass 1 and
// for seg 0.  Under RUNERR, 12 threads draw the run's (S, b_run) of both sensors into rerr, one pair each.
template <bool TERMS, bool RUNERR, int C>
__device__ __forceinline__ NoiseCta noise_prologue(const NoiseParams& p, const NoiseTerms* x, const RunErrs* re,
                                                   int pass, double (*apow)[6], double (*rerr)[12],
                                                   double (&phase)[3], double (&carry)[C]) {
  NoiseCta cta;
  const int segs = (pass == 1) ? p.nseg - 1 : p.nseg;
  cta.run = blockIdx.x / segs;
  cta.seg = static_cast<int>(blockIdx.x % segs);
  cta.seg_hi = min64(p.n, (cta.seg + 1) * p.seg_len);
  cta.seg_lo = (pass == 1) ? cta.seg_hi - p.pass1_len : cta.seg * p.seg_len;
  const int64_t grun = p.run_offset + cta.run;
  cta.run_lo = static_cast<uint32_t>(grun);
  cta.run_hi = static_cast<uint32_t>(grun >> 32);
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
      phase[c] = (uniform01(0xFFFFFFFFu, kDrawPhase + c, cta.run_lo, cta.run_hi, p.k0, p.k1) * 2.0) * kPi;
  }
  const int64_t at = (cta.run * p.nseg + cta.seg) * 6;
#pragma unroll
  for (int c = 0; c < 6; ++c) carry[c] = 0.0;
  if (pass == 0 && p.seg_carry) {
#pragma unroll
    for (int c = 0; c < 6; ++c) carry[c] = p.seg_carry[at + c];
  }
  if constexpr (TERMS) {
#pragma unroll
    for (int c = 0; c < 6; ++c) carry[6 + c] = (pass == 0 && x->seg_carry) ? x->seg_carry[at + c] : 0.0;
  }
  if constexpr (RUNERR) {
    if (tid < 12) run_err_pair(re->s[tid / 6], tid / 6, tid % 6, cta.run_lo, cta.run_hi, p.k0, p.k1, rerr[tid / 6]);
  }
  __syncthreads();
  return cta;
}

// One tile of a K1 or K9 CTA, its samples tile0 .. tile0 + cnt - 1, up to the end of the scan.  The thread makes
// its stretch (the kNoisePer consecutive samples tid kNoisePer ..) one sensor triad at a time (three Box-Muller
// chains in flight) into stage[sensor][sample * 3 + axis]: each measurement without the drift (and walk) at the
// stretch start.  Then the affine scan over the threads, (A, E) o (A', E') = (A A', A' E + E'), leaves in S the
// drift (and under TERMS the walk) at the stretch start, and advances carry to the next tile.  Returns the
// stretch's live samples.  In K1's pass 1 only the drift and the walk advance.
template <bool TERMS, bool RUNERR, int C>
__device__ __forceinline__ int noise_tile(const NoiseParams& p, const NoiseTerms* x, const NoiseCta& cta,
                                          const double (&phase)[3], const double (*apow)[6],
                                          const double (*rerr)[12], double (*stage)[kNoiseTile * 3],
                                          double (*wtot)[kNoiseWarps][2], int64_t tile0, int cnt, int pass,
                                          double (&carry)[C], double (&S)[C]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double r[C];
#pragma unroll
  for (int c = 0; c < C; ++c) r[c] = 0.0;
  int mine = cnt - tid * kNoisePer;                 // live samples of this thread's stretch
  mine = mine < 0 ? 0 : (mine > kNoisePer ? kNoisePer : mine);
  double qe[TERMS ? 6 : 1];                         // TERMS: the quantisation error e[t] of each channel
  if constexpr (TERMS) {
    if (mine > 0 && pass == 0) {
      const uint32_t t0 = static_cast<uint32_t>(tile0 + tid * kNoisePer);
#pragma unroll
      for (int c = 0; c < 6; ++c)
        qe[c] = x->q[c] != 0.0
                    ? x->q[c] * (uniform01(t0, kDrawQuant + c, cta.run_lo, cta.run_hi, p.k0, p.k1) - 0.5)
                    : 0.0;
    }
  }
#pragma unroll 1
  for (int q = 0; q < mine; ++q) {
    const int el = tid * kNoisePer + q;
    const int64_t t = tile0 + el;
    double m3[3];
    triad_sample<0>(p, p.accel, p.ref_accel + t * 3, static_cast<uint32_t>(t), cta.run_lo, cta.run_hi, cta.run,
                    phase, pass == 1, r, m3);
    if constexpr (TERMS) terms_sample<0>(p, *x, t, cta.run_lo, cta.run_hi, pass == 1, r + 6, qe, m3);
    if constexpr (RUNERR) {
      if (pass == 0) run_err_add(rerr[0], p.ref_accel + t * 3, m3);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) stage[0][el * 3 + c] = m3[c];
    triad_sample<1>(p, p.gyro, p.ref_gyro + t * 3, static_cast<uint32_t>(t), cta.run_lo, cta.run_hi, cta.run,
                    phase, pass == 1, r + 3, m3);
    if constexpr (TERMS) terms_sample<1>(p, *x, t, cta.run_lo, cta.run_hi, pass == 1, r + 9, qe + 3, m3);
    if constexpr (RUNERR) {
      if (pass == 0) run_err_add(rerr[1], p.ref_gyro + t * 3, m3);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) stage[1][el * 3 + c] = m3[c];
  }
  double sA[C], sE[C];
#pragma unroll
  for (int c = 0; c < C; ++c) {
    sA[c] = c < 6 ? apow[mine][c] : 1.0;
    sE[c] = r[c];
  }
  affine_scan_warp<C, kNoiseWarps>(sA, sE, wtot, lane, warp);
  __syncthreads();   // warp totals; the staged tile is complete
  affine_scan_block<C, kNoiseWarps>(sA, sE, wtot, lane, warp, carry, S);
  return mine;
}

// K1's body.  TERMS adds the IEEE Std 952 terms of x (DESIGN.md section 4): the rate random walk k runs as six
// more channels of the affine scan with A = 1, the quantisation error carries e[t+1] along the thread's stretch
// (one extra uniform at its start), the rate ramp is R t dt.  RUNERR adds the run-to-run errors of re: the CTA's
// run makes its (S, b_run) of both sensors in the prologue into shared memory (12 threads, one pair each), and
// every triad gets delta = b_run + S ref from there; it has no state in time, so segments carry nothing for it.
// Without TERMS and RUNERR this is K1 as it always was.
template <bool TERMS, bool RUNERR>
__device__ __forceinline__ void imu_noise_body(const NoiseParams& p, const NoiseTerms* x, const RunErrs* re) {
  constexpr int C = TERMS ? 12 : 6;               // scanned channels: drift (accel, gyro), then the walk
  __shared__ double stage[2][kNoiseTile * 3];     // accel, gyro of the tile, [sample][axis]
  __shared__ double wtot[C][kNoiseWarps][2];      // (A, E) of every warp's stretch, per channel
  __shared__ double apow[kNoisePer + 1][6];       // a^q per channel
  __shared__ double rerr[RUNERR ? 2 : 1][12];     // RUNERR: (S row-major, b_run) of accel, gyro for this run
  const int tid = threadIdx.x;
  double phase[3], carry[C];                      // carry: d (and k) at the first sample of the tile
  const NoiseCta cta = noise_prologue<TERMS, RUNERR>(p, x, re, p.pass, apow, rerr, phase, carry);

  for (int64_t tile0 = cta.seg_lo; tile0 < cta.seg_hi; tile0 += kNoiseTile) {
    const int cnt = static_cast<int>(min64(kNoiseTile, cta.seg_hi - tile0));
    double S[C];       // drift (and walk) at the first sample of this thread's stretch
    const int mine =
        noise_tile<TERMS, RUNERR>(p, x, cta, phase, apow, rerr, stage, wtot, tile0, cnt, p.pass, carry, S);
    if (p.pass == 0) {
      // ---- + a^q S on the thread's own samples, then the tile leaves in the caller's layout -------
#pragma unroll 1
      for (int q = 0; q < mine; ++q) {
        const int el = tid * kNoisePer + q;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          stage[0][el * 3 + c] += apow[q][c] * S[c];
          stage[1][el * 3 + c] += apow[q][3 + c] * S[3 + c];
          if constexpr (TERMS) {      // the walk at the stretch start
            stage[0][el * 3 + c] += S[6 + c];
            stage[1][el * 3 + c] += S[9 + c];
          }
        }
      }
      __syncthreads();
      const int64_t base = cta.run * p.osr + tile0 * p.ost;
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
          double* zd = p.z_dump + (cta.run * p.n + t) * 12;
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            const uint32_t t32 = static_cast<uint32_t>(t);
            const Normal2 za = normal_pair(t32, kDrawAccel + c, cta.run_lo, cta.run_hi, p.k0, p.k1);
            const Normal2 zg = normal_pair(t32, kDrawGyro + c, cta.run_lo, cta.run_hi, p.k0, p.k1);
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
    for (int c = 0; c < 6; ++c) p.seg_end[(cta.run * p.nseg + cta.seg) * 6 + c] = carry[c];
    if constexpr (TERMS) {
#pragma unroll
      for (int c = 0; c < 6; ++c) x->seg_end[(cta.run * p.nseg + cta.seg) * 6 + c] = carry[6 + c];
    }
  }
}

__global__ void __launch_bounds__(kNoiseThreads, 4) imu_noise_kernel(const __grid_constant__ NoiseParams p) {
  imu_noise_body<false, false>(p, nullptr, nullptr);
}

__global__ void __launch_bounds__(kNoiseThreads, 3) imu_noise_ex_kernel(const __grid_constant__ NoiseParams p,
                                                                      const __grid_constant__ NoiseTerms x) {
  imu_noise_body<true, false>(p, &x, nullptr);
}

// K1-rx: the run-to-run errors alone, and with the IEEE Std 952 terms
__global__ void __launch_bounds__(kNoiseThreads, 4) imu_noise_rx_kernel(const __grid_constant__ NoiseParams p,
                                                                      const __grid_constant__ RunErrs re) {
  imu_noise_body<false, true>(p, nullptr, &re);
}

__global__ void __launch_bounds__(kNoiseThreads, 3) imu_noise_ex_rx_kernel(const __grid_constant__ NoiseParams p,
                                                                         const __grid_constant__ NoiseTerms x,
                                                                         const __grid_constant__ RunErrs re) {
  imu_noise_body<true, true>(p, &x, &re);
}

// the run-error table: one thread per (run, sensor) writes out[run][sensor][12] = (S row-major, b_run)
__global__ void imu_run_err_kernel(const __grid_constant__ RunErrs re, int64_t runs, int64_t run_offset, uint32_t k0,
                                   uint32_t k1, double* out) {
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= runs * 2) return;
  const int sensor = static_cast<int>(idx % 2);
  const int64_t grun = run_offset + idx / 2;
  const uint32_t run_lo = static_cast<uint32_t>(grun), run_hi = static_cast<uint32_t>(grun >> 32);
  for (int j = 0; j < 6; ++j) run_err_pair(re.s[sensor], sensor, j, run_lo, run_hi, k0, k1, out + idx * 12);
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
