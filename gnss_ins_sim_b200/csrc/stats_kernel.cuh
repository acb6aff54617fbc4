// K3: ensemble error statistics over runs -- InsDataMgr.__array_stats
// (ins_data_manager.py:797-808): max|e|, mean, std (ddof 0, two-pass like np.std).
// Deterministic two-stage reductions (no floating-point atomics): stage 1 writes one
// partial per block, stage 2 (one block) folds them in a fixed order.
// Non-finite errors come out as NumPy's: a NaN sample makes max NaN (max_or_nan,
// max_nan), and the two passes make mean and std NaN or +-inf exactly where
// np.average and np.std do.  No runs (K3x with every shard empty): NaN statistics.
#pragma once
#include "common.cuh"

namespace b2ins {

constexpr int kStatBlocks = 128;   // stage-1 grid
constexpr int kStatMaxComp = 32;

__host__ __device__ inline int stat_threads(int ncomp) { return ncomp * (1024 / ncomp >= 32 ? 32 : 1024 / ncomp); }

// The per-sample loops keep fmax (one instruction on the loop-carried max) and note a
// NaN sample in a flag beside it; the thread's partial max is then NaN, and the folds
// (max_nan) keep it.
__device__ __forceinline__ double max_or_nan(double mx, bool nan) {
  return nan ? __longlong_as_double(0x7ff8000000000000LL) : mx;
}

// MODE 0: sum e and max|e| ; MODE 1: sum (e - mean)^2
template <int MODE>
__global__ void err_stage1_kernel(int64_t runs, int ncomp, const double* __restrict__ err,
                                  const double* __restrict__ mean, double* __restrict__ ws) {
  extern __shared__ double sh[];  // [threads] sums, [threads] maxes
  const int threads = blockDim.x;
  const int c = threadIdx.x % ncomp;   // blockDim.x and the grid stride are multiples of ncomp
  const int64_t total = runs * ncomp;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * threads;
  double acc = 0.0, mx = 0.0;
  bool nan = false;
  const double mu = (MODE == 1) ? mean[c] : 0.0;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * threads + threadIdx.x; i < total; i += stride) {
    const double e = err[i];
    if (MODE == 0) {
      acc += e;
      mx = fmax(mx, fabs(e));
      nan |= e != e;
    } else {
      const double d = e - mu;
      acc += d * d;
    }
  }
  sh[threadIdx.x] = acc;
  sh[threads + threadIdx.x] = max_or_nan(mx, nan);
  __syncthreads();
  if (threadIdx.x < ncomp) {
    double s = 0.0, m = 0.0;
    for (int k = threadIdx.x; k < threads; k += ncomp) {
      s += sh[k];
      m = max_nan(m, sh[threads + k]);
    }
    ws[(static_cast<int64_t>(blockIdx.x) * 2) * ncomp + c] = s;
    ws[(static_cast<int64_t>(blockIdx.x) * 2 + 1) * ncomp + c] = m;
  }
}

// fold the per-block partials: out[0..ncomp) = sum, out[ncomp..2ncomp) = max (MODE 0 only)
template <int MODE>
__global__ void err_stage2_kernel(int nblocks, int ncomp, const double* __restrict__ ws,
                                  double* __restrict__ out) {
  const int c = threadIdx.x;
  if (c >= ncomp) return;
  double s = 0.0, m = 0.0;
  for (int b = 0; b < nblocks; ++b) {
    s += ws[(static_cast<int64_t>(b) * 2) * ncomp + c];
    m = max_nan(m, ws[(static_cast<int64_t>(b) * 2 + 1) * ncomp + c]);
  }
  out[c] = s;
  if (MODE == 0) out[ncomp + c] = m;
}

// single-shard finalisation helpers
__global__ void stats_mean_kernel(int64_t runs, int ncomp, const double* __restrict__ partial,
                                  double* __restrict__ stats) {
  const int c = threadIdx.x;
  if (c >= ncomp) return;
  stats[c] = partial[ncomp + c];                                  // max|e|
  stats[ncomp + c] = partial[c] / static_cast<double>(runs);      // mean
}
__global__ void stats_std_kernel(int64_t runs, int ncomp, const double* __restrict__ partial2,
                                 double* __restrict__ stats) {
  const int c = threadIdx.x;
  if (c >= ncomp) return;
  stats[2 * ncomp + c] = sqrt(partial2[c] / static_cast<double>(runs));
}

// Small ensembles (runs * ncomp <= kStatSmallMax): everything in ONE block and one launch --
// sum/max, mean, second pass, std -- with the same fixed-order folding as the staged path.
constexpr int kStatSmallMax = 1 << 17;
constexpr int kStatSmallThreads = 1024;

__global__ void __launch_bounds__(kStatSmallThreads)
stats_small_kernel(int64_t runs, int ncomp, const double* __restrict__ err, double* __restrict__ stats) {
  __shared__ double sh[2 * kStatSmallThreads];
  __shared__ double mean_sh[kStatMaxComp];
  const int threads = (kStatSmallThreads / ncomp) * ncomp;   // a multiple of ncomp
  const int c = threadIdx.x % ncomp;
  const int64_t total = runs * ncomp;
  const bool on = threadIdx.x < threads;
  double acc = 0.0, mx = 0.0;
  bool nan = false;
  if (on)
    for (int64_t i = threadIdx.x; i < total; i += threads) {
      const double e = err[i];
      acc += e;
      mx = fmax(mx, fabs(e));
      nan |= e != e;
    }
  sh[threadIdx.x] = acc;
  sh[kStatSmallThreads + threadIdx.x] = max_or_nan(mx, nan);
  __syncthreads();
  if (threadIdx.x < ncomp) {
    double s = 0.0, m = 0.0;
    for (int k = threadIdx.x; k < threads; k += ncomp) {
      s += sh[k];
      m = max_nan(m, sh[kStatSmallThreads + k]);
    }
    stats[c] = m;
    const double mean = s / static_cast<double>(runs);
    stats[ncomp + c] = mean;
    mean_sh[c] = mean;
  }
  __syncthreads();
  const double mu = mean_sh[c];
  acc = 0.0;
  if (on)
    for (int64_t i = threadIdx.x; i < total; i += threads) {
      const double d = err[i] - mu;
      acc += d * d;
    }
  sh[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x < ncomp) {
    double s = 0.0;
    for (int k = threadIdx.x; k < threads; k += ncomp) s += sh[k];
    stats[2 * ncomp + c] = sqrt(s / static_cast<double>(runs));
  }
}

// ---- K3x: statistics fused with their exchange over NVLink peer memory ---------------------
// Multi-GPU ensembles: instead of K3 followed by an NCCL collective, ONE kernel per rank computes
// the shard statistics, stores (max, mean, std, count) straight into every peer's receive
// window through peer-mapped (symmetric) memory, raises a flag with a system-scope release
// store, waits for the other ranks' flags and merges all shards with Chan's update.  The payload
// is 29 doubles per rank; what is saved is the collective's launch + host round trips.
constexpr int kXchgSlot = 32;       // doubles per (parity, source rank): 3*9 stats, count, flag
constexpr int kXchgMaxWorld = 16;

struct XchgParams {
  int64_t runs;
  int ncomp, rank, world;
  uint64_t seq;                      // call counter >= 1; windows are double-buffered on seq & 1
  const double* err;
  double* peer[kXchgMaxWorld];       // peer[p]: rank p's window [2][world][kXchgSlot], mapped here
  double* out;                       // [3][ncomp] merged statistics
  int* timeout_flag;                 // set to 1 if a peer never showed up
};

__global__ void __launch_bounds__(kStatSmallThreads)
stats_exchange_kernel(const __grid_constant__ XchgParams p) {
  __shared__ double sh[2 * kStatSmallThreads];
  __shared__ double loc[3 * kStatMaxComp + 1];
  __shared__ int arrived[kXchgMaxWorld];   // 0: the peer's slot still holds an older call's values
  const int nc = p.ncomp;
  const int threads = (kStatSmallThreads / nc) * nc;
  const int c = threadIdx.x % nc;
  const int64_t total = p.runs * nc;
  const bool on = threadIdx.x < threads;
  // ---- local (max, mean, std): same two passes as stats_small_kernel -------------------------
  double acc = 0.0, mx = 0.0;
  bool nan = false;
  if (on)
    for (int64_t i = threadIdx.x; i < total; i += threads) {
      const double e = p.err[i];
      acc += e;
      mx = fmax(mx, fabs(e));
      nan |= e != e;
    }
  sh[threadIdx.x] = acc;
  sh[kStatSmallThreads + threadIdx.x] = max_or_nan(mx, nan);
  __syncthreads();
  if (threadIdx.x < nc) {
    double s = 0.0, m = 0.0;
    for (int k = threadIdx.x; k < threads; k += nc) {
      s += sh[k];
      m = max_nan(m, sh[kStatSmallThreads + k]);
    }
    loc[c] = m;
    loc[nc + c] = p.runs > 0 ? s / static_cast<double>(p.runs) : 0.0;
  }
  __syncthreads();
  const double mu = loc[nc + c];
  acc = 0.0;
  if (on)
    for (int64_t i = threadIdx.x; i < total; i += threads) {
      const double d = p.err[i] - mu;
      acc += d * d;
    }
  sh[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x < nc) {
    double s = 0.0;
    for (int k = threadIdx.x; k < threads; k += nc) s += sh[k];
    loc[2 * nc + c] = p.runs > 0 ? sqrt(s / static_cast<double>(p.runs)) : 0.0;
  }
  if (threadIdx.x == 0) loc[3 * nc] = static_cast<double>(p.runs);
  __syncthreads();
  // ---- push to every rank's window (peer stores over NVLink), then the flags ------------------
  const int par = static_cast<int>(p.seq & 1);
  const int64_t slot = (static_cast<int64_t>(par) * p.world + p.rank) * kXchgSlot;
  if (threadIdx.x <= 3 * nc) {
    const double v = loc[threadIdx.x];
    for (int q = 0; q < p.world; ++q) p.peer[q][slot + threadIdx.x] = v;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x < p.world) {
    unsigned long long* f = reinterpret_cast<unsigned long long*>(p.peer[threadIdx.x] + slot + kXchgSlot - 1);
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(f), "l"(p.seq) : "memory");
    // ---- wait for rank threadIdx.x's contribution in MY window -------------------------------
    const unsigned long long* mine = reinterpret_cast<const unsigned long long*>(
        p.peer[p.rank] + (static_cast<int64_t>(par) * p.world + threadIdx.x) * kXchgSlot + kXchgSlot - 1);
    unsigned long long seen = 0;
    const long long t0 = clock64();
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(mine) : "memory");
      if (clock64() - t0 > 40000000000LL) {   // ~20 s: a peer never launched
        *p.timeout_flag = 1;
        break;
      }
    } while (seen < p.seq);
    arrived[threadIdx.x] = seen >= p.seq;   // a stale slot (an older call's statistics) is never merged
  }
  __syncthreads();
  // ---- Chan merge of all shards, one thread per component, fixed rank order -------------------
  if (threadIdx.x < nc) {
    const double* win = p.peer[p.rank] + static_cast<int64_t>(par) * p.world * kXchgSlot;
    double n_a = 0.0, mx_a = 0.0, mean_a = 0.0, m2_a = 0.0;
    for (int q = 0; q < p.world; ++q) {
      const double* sl = win + static_cast<int64_t>(q) * kXchgSlot;
      const double n_b = sl[3 * nc];
      if (n_b <= 0.0 || !arrived[q]) continue;
      const double mean_b = sl[nc + c], std_b = sl[2 * nc + c];
      const double m2_b = std_b * std_b * n_b;
      if (n_a == 0.0) {
        n_a = n_b; mx_a = sl[c]; mean_a = mean_b; m2_a = m2_b;
      } else {
        const double n = n_a + n_b, delta = mean_b - mean_a;
        mean_a = mean_step(mean_a, mean_b, delta, n_b / n);
        m2_a += m2_b + delta * delta * (n_a * n_b / n);
        mx_a = max_nan(mx_a, sl[c]);
        n_a = n;
      }
    }
    const double none = __longlong_as_double(0x7ff8000000000000LL);   // no runs on any rank
    p.out[c] = n_a > 0.0 ? mx_a : none;
    p.out[nc + c] = n_a > 0.0 ? mean_a : none;
    p.out[2 * nc + c] = n_a > 0.0 ? sqrt(m2_a / n_a) : none;
  }
}

}  // namespace b2ins
