// K9: per-run error statistics of the IMU measurements, reduced inside the noise generator, and K3p:
// per-run error statistics of a materialised per-run array (magnetometer, GPS).  Both compute what
// InsDataMgr.get_error_stats does for sensor data (ins_data_manager.py:524-541, :717-808): the error
// e = meas - ref, its value at the last sample, and over the samples from a start index max|e|, mean
// and std (ddof 0).
//
// K9 has K1's launch shape (one CTA per (run, time segment), 896-sample tiles; the segmented form's pass 1
// and noise_carry_kernel are K1's own) and runs K1's generator: noise_prologue, then for every tile
// noise_tile (the stretch loop and the affine Gauss-Markov scan over the threads).  The finished tile is
// reduced instead of stored: nothing of the series leaves the SM.
//
// Determinism: every reduction runs in a fixed order, with no floating-point atomics.  A thread reduces
// its own stretch of a tile in two passes (sum and max, then the squared deviations from the stretch
// mean) and merges the result into its running (count, mean, M2, max) with Chan's update; the 128
// thread partials are merged by a fixed shuffle tree and the four warp totals in warp order; time
// segments are merged in segment order by err_stats_fold_kernel.
//
// Non-finite errors come out as NumPy's: max_nan keeps a NaN, mean_step carries a +-inf or NaN mean through
// the merges, and the M2 of any stretch with a non-finite sample is NaN, so std is NaN there as np.std's is.
#pragma once
#include "noise_kernel.cuh"

namespace b2ins {

constexpr int kErrCh = 6;                        // accel x y z, gyro x y z (K1's channel order)
constexpr int kErrPartial = 1 + 3 * kErrCh;      // count, mean[6], M2[6], max|e|[6]

struct ErrStatsParams {
  NoiseParams np;          // the generator (pass 0); its output pointers are unused
  int64_t stats_start;     // first sample of the process statistics; < 0: end_err only
  double* end_err;         // [runs][6]
  double* proc_stats;      // [runs][3][6] max|e|, mean, std (written here when nseg == 1)
  double* partial;         // [runs][nseg][kErrPartial] (nseg > 1)
};

// (na, ma, m2a, xa) <- (na, ma, m2a, xa) (+) (nb, mb, m2b, xb)  (Chan, Golub, LeVeque)
__device__ __forceinline__ void chan_merge(double& na, double& ma, double& m2a, double& xa, double nb, double mb,
                                           double m2b, double xb) {
  if (nb == 0.0) return;
  if (na == 0.0) {
    na = nb;
    ma = mb;
    m2a = m2b;
    xa = xb;
    return;
  }
  const double n = na + nb, d = mb - ma, f = nb / n;
  ma = mean_step(ma, mb, d, f);
  m2a += m2b + d * d * (na * f);
  xa = max_nan(xa, xb);
  na = n;
}

// the statistics of no samples (n = 0) are NaN
__device__ __forceinline__ void write_stats(double* ps, int c, int nc, double n, double mean, double m2, double mx) {
  const double none = __longlong_as_double(0x7ff8000000000000LL);
  ps[c] = n > 0.0 ? mx : none;
  ps[nc + c] = n > 0.0 ? mean : none;
  ps[2 * nc + c] = n > 0.0 ? sqrt(m2 / n) : none;
}

// K9's body; TERMS: with the IEEE Std 952 terms of x, RUNERR: with the run-to-run errors of re, generated as K1's
// imu_noise_body<TERMS, RUNERR> makes them
template <bool TERMS, bool RUNERR>
__device__ __forceinline__ void imu_err_stats_body(const ErrStatsParams& P, const NoiseTerms* x, const RunErrs* re) {
  constexpr int C = TERMS ? 12 : 6;
  const NoiseParams& p = P.np;
  __shared__ double stage[2][kNoiseTile * 3];     // accel, gyro of the tile, [sample][axis]
  __shared__ double wtot[C][kNoiseWarps][2];
  __shared__ double apow[kNoisePer + 1][6];
  __shared__ double rerr[RUNERR ? 2 : 1][12];     // RUNERR: (S row-major, b_run) of accel, gyro for this run
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool want_stats = P.stats_start >= 0;
  double an = 0.0, am[6], a2[6], ax[6];           // the thread's running statistics
#pragma unroll
  for (int c = 0; c < 6; ++c) am[c] = a2[c] = ax[c] = 0.0;
  double phase[3], carry[C];
  const NoiseCta cta = noise_prologue<TERMS, RUNERR>(p, x, re, 0, apow, rerr, phase, carry);

  for (int64_t tile0 = cta.seg_lo; tile0 < cta.seg_hi; tile0 += kNoiseTile) {
    const int cnt = static_cast<int>(min64(kNoiseTile, cta.seg_hi - tile0));
    double S[C];
    const int mine = noise_tile<TERMS, RUNERR>(p, x, cta, phase, apow, rerr, stage, wtot, tile0, cnt, 0, carry, S);
    // ---- the thread's own samples: the measurement exactly as K1 stores it, minus the truth --------
    // pass A: e (kept in the stage), the end-point error, sum and max over the samples >= stats_start
    const int64_t t_lo = tile0 + tid * kNoisePer;
    int q0 = 0;
    if (want_stats && P.stats_start > t_lo) q0 = P.stats_start - t_lo > mine ? mine : static_cast<int>(P.stats_start - t_lo);
    double bs[6], bx[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) bs[c] = bx[c] = 0.0;
#pragma unroll 1
    for (int q = 0; q < mine; ++q) {
      const int el = tid * kNoisePer + q;
      const int64_t t = tile0 + el;
      double e[6];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        double ma = fma(apow[q][c], S[c], stage[0][el * 3 + c]);
        double mg = fma(apow[q][3 + c], S[3 + c], stage[1][el * 3 + c]);
        if constexpr (TERMS) {      // the walk at the stretch start
          ma += S[6 + c];
          mg += S[9 + c];
        }
        e[c] = ma - p.ref_accel[t * 3 + c];
        e[3 + c] = mg - p.ref_gyro[t * 3 + c];
        stage[0][el * 3 + c] = e[c];
        stage[1][el * 3 + c] = e[3 + c];
      }
      if (t == p.n - 1) {
#pragma unroll
        for (int c = 0; c < 6; ++c) P.end_err[cta.run * kErrCh + c] = e[c];
      }
      if (q >= q0) {
#pragma unroll
        for (int c = 0; c < 6; ++c) {
          bs[c] += e[c];
          bx[c] = max_nan(bx[c], fabs(e[c]));
        }
      }
    }
    const int k = want_stats ? mine - q0 : 0;
    if (k > 0) {
      // pass B: squared deviations from the stretch mean, then Chan into the running statistics
      const double kn = static_cast<double>(k);
      double bm[6], b2[6];
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        bm[c] = bs[c] / kn;
        b2[c] = 0.0;
      }
#pragma unroll 1
      for (int q = q0; q < mine; ++q) {
        const int el = tid * kNoisePer + q;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const double da = stage[0][el * 3 + c] - bm[c], dg = stage[1][el * 3 + c] - bm[3 + c];
          b2[c] = fma(da, da, b2[c]);
          b2[3 + c] = fma(dg, dg, b2[3 + c]);
        }
      }
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        double n0 = an;
        chan_merge(n0, am[c], a2[c], ax[c], kn, bm[c], b2[c], bx[c]);
      }
      an += kn;
    }
    __syncthreads();   // the stage and the warp totals are rewritten by the next tile
  }
  if (!want_stats) return;
  // ---- the CTA's statistics: a fixed shuffle tree within each warp, then the warps in order ---------
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const double nb = __shfl_down_sync(0xffffffffu, an, off);
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      const double mb = __shfl_down_sync(0xffffffffu, am[c], off);
      const double m2b = __shfl_down_sync(0xffffffffu, a2[c], off);
      const double xb = __shfl_down_sync(0xffffffffu, ax[c], off);
      double n0 = an;
      if (lane + off < 32) chan_merge(n0, am[c], a2[c], ax[c], nb, mb, m2b, xb);
    }
    if (lane + off < 32) an += nb;
  }
  double* red = &stage[0][0];                     // [warp][kErrPartial]
  if (lane == 0) {
    red[warp * kErrPartial] = an;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      red[warp * kErrPartial + 1 + c] = am[c];
      red[warp * kErrPartial + 7 + c] = a2[c];
      red[warp * kErrPartial + 13 + c] = ax[c];
    }
  }
  __syncthreads();
  if (tid < kErrCh) {
    const int c = tid;
    double n = 0.0, m = 0.0, m2 = 0.0, mx = 0.0;
    for (int w = 0; w < kNoiseWarps; ++w)
      chan_merge(n, m, m2, mx, red[w * kErrPartial], red[w * kErrPartial + 1 + c], red[w * kErrPartial + 7 + c],
                 red[w * kErrPartial + 13 + c]);
    if (p.nseg == 1) {
      write_stats(P.proc_stats + cta.run * 3 * kErrCh, c, kErrCh, n, m, m2, mx);
    } else {
      double* o = P.partial + (cta.run * p.nseg + cta.seg) * kErrPartial;
      if (c == 0) o[0] = n;
      o[1 + c] = m;
      o[7 + c] = m2;
      o[13 + c] = mx;
    }
  }
}

__global__ void __launch_bounds__(kNoiseThreads, 4) imu_err_stats_kernel(const __grid_constant__ ErrStatsParams P) {
  imu_err_stats_body<false, false>(P, nullptr, nullptr);
}

__global__ void __launch_bounds__(kNoiseThreads, 3) imu_err_stats_ex_kernel(const __grid_constant__ ErrStatsParams P,
                                                                          const __grid_constant__ NoiseTerms x) {
  imu_err_stats_body<true, false>(P, &x, nullptr);
}

// K9-rx: the run-to-run errors alone, and with the IEEE Std 952 terms
__global__ void __launch_bounds__(kNoiseThreads, 4) imu_err_stats_rx_kernel(const __grid_constant__ ErrStatsParams P,
                                                                          const __grid_constant__ RunErrs re) {
  imu_err_stats_body<false, true>(P, nullptr, &re);
}

__global__ void __launch_bounds__(kNoiseThreads, 3)
    imu_err_stats_ex_rx_kernel(const __grid_constant__ ErrStatsParams P, const __grid_constant__ NoiseTerms x,
                               const __grid_constant__ RunErrs re) {
  imu_err_stats_body<true, true>(P, &x, &re);
}

// the segments of every run, merged in segment order: one thread per (run, channel)
__global__ void err_stats_fold_kernel(const __grid_constant__ ErrStatsParams P) {
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= P.np.runs * kErrCh) return;
  const int64_t run = idx / kErrCh;
  const int c = static_cast<int>(idx % kErrCh);
  double n = 0.0, m = 0.0, m2 = 0.0, mx = 0.0;
  for (int s = 0; s < P.np.nseg; ++s) {
    const double* o = P.partial + (run * P.np.nseg + s) * kErrPartial;
    chan_merge(n, m, m2, mx, o[0], o[1 + c], o[7 + c], o[13 + c]);
  }
  write_stats(P.proc_stats + run * 3 * kErrCh, c, kErrCh, n, m, m2, mx);
}

// ---- K3p: x [runs][m][nc] against a shared ref [m][nc] --------------------------------------------
constexpr int kProcThreads = 256;
constexpr int kProcMaxComp = 8;

// One CTA per run.  Thread i takes rows i, i + 256, ... (consecutive threads, consecutive rows) and keeps
// Welford statistics of them; the 256 partials are merged by the same fixed tree as K9's.
__global__ void __launch_bounds__(kProcThreads) proc_stats_kernel(int64_t m, int nc, const double* __restrict__ x,
                                                                  const double* __restrict__ ref, int64_t start,
                                                                  double* __restrict__ end_err,
                                                                  double* __restrict__ proc_stats) {
  __shared__ double red[kProcThreads / 32][1 + 3 * kProcMaxComp];
  const int64_t run = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double* xr = x + run * m * nc;
  double an = 0.0, am[kProcMaxComp], a2[kProcMaxComp], ax[kProcMaxComp];
#pragma unroll
  for (int c = 0; c < kProcMaxComp; ++c) am[c] = a2[c] = ax[c] = 0.0;
  for (int64_t i = start + tid; i < m; i += kProcThreads) {
    an += 1.0;
    const double inv = 1.0 / an;
#pragma unroll
    for (int c = 0; c < kProcMaxComp; ++c) {
      if (c < nc) {
        const double e = xr[i * nc + c] - ref[i * nc + c];
        const double d = e - am[c];
        am[c] = mean_step(am[c], e, d, inv);
        a2[c] = fma(d, e - am[c], a2[c]);
        ax[c] = max_nan(ax[c], fabs(e));
      }
    }
  }
  if (tid == 0 && end_err && m > 0) {
    for (int c = 0; c < nc; ++c) end_err[run * nc + c] = xr[(m - 1) * nc + c] - ref[(m - 1) * nc + c];
  }
  if (!proc_stats) return;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const double nb = __shfl_down_sync(0xffffffffu, an, off);
#pragma unroll
    for (int c = 0; c < kProcMaxComp; ++c) {
      const double mb = __shfl_down_sync(0xffffffffu, am[c], off);
      const double m2b = __shfl_down_sync(0xffffffffu, a2[c], off);
      const double xb = __shfl_down_sync(0xffffffffu, ax[c], off);
      double n0 = an;
      if (lane + off < 32) chan_merge(n0, am[c], a2[c], ax[c], nb, mb, m2b, xb);
    }
    if (lane + off < 32) an += nb;
  }
  if (lane == 0) {
    red[warp][0] = an;
#pragma unroll
    for (int c = 0; c < kProcMaxComp; ++c) {
      red[warp][1 + c] = am[c];
      red[warp][1 + kProcMaxComp + c] = a2[c];
      red[warp][1 + 2 * kProcMaxComp + c] = ax[c];
    }
  }
  __syncthreads();
  if (tid < nc) {
    const int c = tid;
    double n = 0.0, mu = 0.0, m2 = 0.0, mx = 0.0;
    for (int w = 0; w < kProcThreads / 32; ++w)
      chan_merge(n, mu, m2, mx, red[w][0], red[w][1 + c], red[w][1 + kProcMaxComp + c],
                 red[w][1 + 2 * kProcMaxComp + c]);
    write_stats(proc_stats + run * 3 * nc, c, nc, n, mu, m2, mx);
  }
}

}  // namespace b2ins
