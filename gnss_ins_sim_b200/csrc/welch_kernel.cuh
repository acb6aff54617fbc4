// K11: Welch power spectral density -- scipy.signal.welch(x, fs, window, nperseg = N, noverlap = D) with
// detrend='constant', scaling='density', average='mean', one-sided, nfft = N:
//
//   S = N - D, K = (n - D) / S segments;  y_j[m] = (x[jS + m] - mean_m x[jS + m]) w[m]
//   psd[k] = (1/K) sum_j c_k |X_j[k]|^2 / (fs sum w^2),  X_j = DFT_N(y_j),  c_0 = c_{L-1} = 1, else 2,
//   k < L = N/2 + 1;  freq[k] = k / (N (1/fs))  (np.fft.rfftfreq, bit for bit)
//
// Transform.  The real length-N DFT is one complex DFT of length M = N/2 (the forward form of K5's packing):
// z_m = y_{2m} + j y_{2m+1}, Z = DFT_M(z), 2 X_k = A_k - j e^{-2 pi j k / N} D_k with A_k = Z_k + conj Z_{M-k},
// D_k = Z_k - conj Z_{M-k} (Z_M = Z_0).  K5's primitives do the work (psd_kernel.cuh): M a power of two takes
// fft_dit on the bit-reversed placement; any other M <= 4096 takes K5's Bluestein pipeline on conj z, whose
// output conjugated is the forward transform times P (K5's chirp transform is reused as it is).
//
// Shape.  A CTA owns one (series, chunk of segments) work item at a time and accumulates c-weighted |2X|^2 in
// registers, bins k = tid / G + r * (512 / G).  Small transforms (P <= 1024) run G = min(32, 1024 / P)
// segments of the chunk side by side in the work array, so every barrier of a stage serves G transforms; the
// G slot sums are added by an xor tree over adjacent lanes at the chunk end.  P up to 8192 (N = 16384) fills
// K5's 192 KB of shared memory with one segment; the window is read through L1/L2.  Consecutive segments of a
// chunk overlap, so their second read of a sample comes from L2.
//
// Mean.  The segment mean is removed as a pair hi + lo: hi is the sum of x 2^-e (2^e >= N) divided by N 2^-e,
// lo the same of the residuals x - hi, and y = ((x - hi) - lo) w.  A one-pass mean carries a rounding of order
// u |mean| into every sample, which leaks u |mean| sum w into bins 0 and 1: 5 % of bin 0 for an offset of 1e4
// under noise of 1e-9.  The pair leaves u^2 |mean| plus the roundings of the residuals, and nothing for a
// constant series (its residuals are exact and lo = (N d 2^-e) / (N 2^-e) = d).
//
// Range.  Every rescaling is a power of two, so the bits are those of the plain formula wherever nothing over-
// or underflows:
//   * the mean sums x 2^-e, and y is formed as ((x 2^-e - hi 2^-e) - lo 2^-e) (w 2^-c), 2^c >= 16 sqrt(sum w^2)
//     (times P^3 more on the Bluestein path): no value of the transform can overflow, so finite samples never
//     give NaN;
//   * re and im are scaled by g = 2^(e+c-a-4) (1/2, or 1/(2P) on the Bluestein path) before squaring, with
//     2^(2a) near fs sum w^2, so |g 2X|^2 is at most 2^-6 of the segment's own PSD;
//   * each power is scaled by 2^-ceil(log2 Q) in a chunk and each chunk sum by 2^-ceil(log2 nchunk) in
//     welch_finish_kernel;
// welch_prep_kernel folds 2^(2a+8), the two chunk factors and 1/4 (1/(4P^2)) into wscale.  A bin is +inf
// where the PSD exceeds DBL_MAX, and below that only where one segment's own PSD exceeds 16 DBL_MAX.  The
// trade-off is at the small end: the scaled terms keep full precision down to a PSD of about
// 2^(-1014 + ceil(log2 Q) + ceil(log2 nchunk)) (1e-300 for every N at up to 2^8 chunks, whatever fs); below
// that they round as subnormals, where the unscaled |2X|^2, about fs sum w^2 times the PSD, kept more bits.
//
// Determinism.  The chunk length Q (segments) depends on N alone and G on N alone, so each series gives the
// same bits whatever the batch, layout or position.  With more than one chunk, welch_finish_kernel adds the
// chunk partials in chunk order.  A NaN or +-inf sample inside a used segment makes its mean non-finite and
// every bin NaN, as scipy gives; samples past the last segment are never read.
#pragma once
#include "psd_kernel.cuh"

namespace b2ins {

constexpr int kWelchThreads = 512;
constexpr int kWelchBatchPoints = 1024;   // complex points per round of the small-transform form
constexpr int kWelchAccLarge = 17;        // ceil(8193 / 512): the bins of N = 16384 over 512 threads
constexpr int kWelchAccSmall = 3;         // G (M + 1) <= 1.5 * 1024 for P <= 1024
constexpr int64_t kWelchChunkSamples = int64_t(1) << 18;

struct WelchPlan {
  int N, M, P, logP, G, bluestein;
  int64_t S, K, Q, nchunk;   // step, segments, segments per chunk, chunks per series
};

// false: N is not a length K11 transforms (even, >= 16, a power of two <= 16384 or at most 8192), or
// D, n do not give a segment
inline bool welch_plan(int64_t n, int64_t N, int64_t D, WelchPlan* w) {
  if (N < 16 || N > 16384 || D < 0 || D >= N || n < N) return false;
  int bluestein = 0;
  const int P = psd_fft_plan(static_cast<int>(N), &bluestein);
  if (P == 0) return false;
  w->N = static_cast<int>(N);
  w->M = w->N / 2;
  w->P = P;
  w->logP = 0;
  while ((1 << w->logP) < P) ++w->logP;
  w->bluestein = bluestein;
  w->G = P <= kWelchBatchPoints ? (kWelchBatchPoints / P < 32 ? kWelchBatchPoints / P : 32) : 1;
  w->S = N - D;
  w->K = (n - D) / w->S;
  const int64_t rounds = kWelchChunkSamples / (static_cast<int64_t>(w->G) * N);
  w->Q = w->G * (rounds > 1 ? rounds : 1);
  w->nchunk = (w->K + w->Q - 1) / w->Q;
  return true;
}

struct WelchParams {
  const double* x;   // series s, sample t: x[s / inner * outer_stride + s % inner + t * sample_stride]
  int64_t inner, outer_stride, sample_stride, nseries;
  int64_t S, K, Q, nchunk;
  int N, M, P, logP, G, bluestein;
  double fs;
  const double* window;   // [N]
  const double2* bhat;    // [P] K5's transform of the conjugate chirp (Bluestein)
  double* wscale;         // [3] set by welch_prep_kernel: the c-free scale of a bin's sum
                          // 2^(2a + 8 + qc + qn) / (K fs sum w^2), g = 2^(e+c-a-4) post, and 2^-c
  double post;            // 1/2, times 1/P on the Bluestein path
  double mean_scale;      // 2^-e, 2^e >= N: the mean's summands and y
  double mean_div;        // N 2^-e
  double chunk_scale;     // 2^-qc, 2^qc >= Q: each power within a chunk
  double part_scale;      // 2^-qn, 2^qn >= nchunk (1 for one chunk): each chunk sum
  double* psd;            // [nseries][M + 1]
  double* part;           // [nseries][nchunk][M + 1] chunk sums (nchunk > 1)
  double* freq;           // [M + 1]
};

// sum of v over the `gsz` consecutive threads of a group (gsz a power of two >= 16), the same bits on every
// thread of the group; red: kWelchThreads / 32 doubles, free until the next barrier
__device__ __forceinline__ double welch_group_sum(double v, int gsz, double* red) {
  for (int o = (gsz < 32 ? gsz : 32) / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (gsz <= 32) return v;
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  const int nw = gsz >> 5, w0 = (static_cast<int>(threadIdx.x) / gsz) * nw;
  double t = red[w0];
  for (int i = 1; i < nw; ++i) t += red[w0 + i];
  return t;
}

// freq and the bin scale, once per launch (one CTA)
__global__ void __launch_bounds__(kWelchThreads) welch_prep_kernel(const __grid_constant__ WelchParams p) {
  __shared__ double red[kWelchThreads / 32];
  double s = 0.0;
  for (int m = threadIdx.x; m < p.N; m += kWelchThreads) s = fma(p.window[m], p.window[m], s);
  s = welch_group_sum(s, kWelchThreads, red);
  if (threadIdx.x == 0) {
    const double f = p.fs * s;
    // 2^(2a) within a factor 4 of fs sum w^2, so |g 2X|^2 is near the bin's power times fs
    int a = (f > 0.0 && isfinite(f)) ? ilogb(f) / 2 : 0;
    a = a < -500 ? -500 : (a > 500 ? 500 : a);
    // 2^-8 more: a segment's term overflows only where it is 64 times the largest finite PSD
    const double back = ldexp(1.0, 2 * a + 8) / (p.chunk_scale * p.part_scale);
    // 2^c >= 16 max |w| (max |w| <= sqrt(sum w^2)); P^3 bounds the Bluestein pipeline's growth over M
    const int c = (s > 0.0 && isfinite(s) ? ilogb(s) / 2 : 0) + 5 + (p.bluestein ? 3 * p.logP : 0);
    const int e = ilogb(1.0 / p.mean_scale);
    p.wscale[0] = back / (static_cast<double>(p.K) * f);
    p.wscale[1] = ldexp(p.post, e + c - a - 4);
    p.wscale[2] = ldexp(1.0, -c);
  }
  const double val = 1.0 / (static_cast<double>(p.N) * (1.0 / p.fs));
  for (int k = threadIdx.x; k <= p.M; k += kWelchThreads) p.freq[k] = static_cast<double>(k) * val;
}

// Z_k of the segment at z (times P on the Bluestein path), k < M
template <bool BLUE>
__device__ __forceinline__ double2 welch_z(const double2* z, int k, const WelchParams& p) {
  if (!BLUE) return z[k];
  const double2 r = cmul(z[bitrev(k, p.logP)], chirp(k, p.M));
  return make_double2(r.x, -r.y);
}

// |g 2 X_k|^2 (g: wscale[1], 1/P of it undoing the Bluestein path's factor P), k <= M;
// tw: e^{2 pi j i / M}, i < M / 2 (radix-2 path)
template <bool BLUE>
__device__ __forceinline__ double welch_bin_power(const double2* z, int k, const WelchParams& p,
                                                  const double2* tw, double2 half_step, double g) {
  const double2 zk = welch_z<BLUE>(z, k == p.M ? 0 : k, p);
  const double2 zc = welch_z<BLUE>(z, k == 0 ? 0 : p.M - k, p);
  const double2 a = make_double2(zk.x + zc.x, zk.y - zc.y);      // Z_k + conj Z_{M-k}
  const double2 d = make_double2(zk.x - zc.x, zk.y + zc.y);      // Z_k - conj Z_{M-k}
  double2 w;                                                      // e^{-pi j k / M}
  if (!BLUE) {
    const int h = k >> 1;
    w = h < p.M / 2 ? make_double2(tw[h].x, -tw[h].y) : make_double2(-1.0, 0.0);
    if (k & 1) w = cmul(w, half_step);
  } else {
    sincospi(-static_cast<double>(k) / static_cast<double>(p.M), &w.y, &w.x);
  }
  const double2 t = cmul(w, make_double2(d.y, -d.x));             // e^{-pi j k / M} (-j D_k)
  const double re = (a.x + t.x) * g, im = (a.y + t.y) * g;
  return fma(re, re, im * im);
}

template <int ACC, bool BLUE>
__global__ void __launch_bounds__(kWelchThreads, 1) welch_kernel(const __grid_constant__ WelchParams p) {
  extern __shared__ __align__(16) unsigned char welch_smem[];
  __shared__ double red[kWelchThreads / 32];
  double2* x = reinterpret_cast<double2*>(welch_smem);   // [G][P]
  double2* tw = x + p.G * p.P;                            // [P / 2]
  fft_twiddles(tw, p.P);
  const int tid = threadIdx.x;
  const int gsz = kWelchThreads / p.G;                    // threads per segment while loading
  const int lg = tid / gsz, lr = tid % gsz;
  const int slot = tid & (p.G - 1);                       // segment slot whose bins this thread sums
  const int kb = tid / p.G, kstep = kWelchThreads / p.G;
  double2 half_step;                                      // e^{-pi j / M}
  sincospi(-1.0 / static_cast<double>(p.M), &half_step.y, &half_step.x);
  const double g = p.wscale[1], wsc = p.wscale[2], ms = p.mean_scale;
  const int L = p.M + 1;
  const int64_t ss = p.sample_stride;
  for (int64_t item = blockIdx.x; item < p.nseries * p.nchunk; item += gridDim.x) {
    const int64_t s = item / p.nchunk, c = item % p.nchunk;
    const double* xs = p.x + (s / p.inner) * p.outer_stride + (s % p.inner);
    const int64_t j0 = c * p.Q, j1 = (j0 + p.Q < p.K) ? j0 + p.Q : p.K;
    double acc[ACC];
#pragma unroll
    for (int r = 0; r < ACC; ++r) acc[r] = 0.0;
    for (int64_t jb = j0; jb < j1; jb += p.G) {
      const bool live = jb + lg < j1;
      const double* seg = xs + (jb + lg) * p.S * ss;
      double2* xg = x + lg * p.P;
      __syncthreads();   // the previous round has left the work array
      double sum = 0.0;
      if (live) {
        for (int m = lr; m < p.M; m += gsz) {
          const double u = seg[(2 * static_cast<int64_t>(m)) * ss], v = seg[(2 * static_cast<int64_t>(m) + 1) * ss];
          xg[bitrev(m, p.logP)] = make_double2(u, v);
          sum += u * ms + v * ms;
        }
      }
      const double hi = welch_group_sum(sum, gsz, red) / p.mean_div;
      double res = 0.0;
      if (live) {
        for (int m = lr; m < p.M; m += gsz) {
          const double2 v = xg[bitrev(m, p.logP)];
          res += (v.x * ms - hi * ms) + (v.y * ms - hi * ms);
        }
      }
      if (gsz > 32) __syncthreads();   // every warp has read red
      const double lo = welch_group_sum(res, gsz, red) / p.mean_div;
      for (int m = lr; m < p.M; m += gsz) {
        const int i = bitrev(m, p.logP);
        const double2 v = live ? xg[i] : make_double2(0.0, 0.0);
        const double2 y = make_double2(((v.x * ms - hi * ms) - lo * ms) * (__ldg(p.window + 2 * m) * wsc),
                                       ((v.y * ms - hi * ms) - lo * ms) * (__ldg(p.window + 2 * m + 1) * wsc));
        xg[i] = BLUE ? cmul(make_double2(y.x, -y.y), chirp(m, p.M)) : y;
      }
      if (BLUE) {
        for (int m = p.M + lr; m < p.P; m += gsz) xg[bitrev(m, p.logP)] = make_double2(0.0, 0.0);
        fft_dit<-1>(x, tw, p.P, p.G);
        for (int i = tid; i < p.G * p.P; i += kWelchThreads) x[i] = cmul(x[i], p.bhat[i & (p.P - 1)]);
        fft_dif<1>(x, tw, p.P, p.G);
      } else {
        fft_dit<-1>(x, tw, p.P, p.G);
      }
      if (jb + slot < j1) {
        const double2* z = x + slot * p.P;
#pragma unroll
        for (int r = 0; r < ACC; ++r) {
          // opaque to the compiler: a bin's addresses and twiddle are the same in every round, and hoisting
          // those of all ACC bins out of the round loop spills the accumulators
          int k = kb + r * kstep;
          asm volatile("" : "+r"(k));
          if (k < L) acc[r] += welch_bin_power<BLUE>(z, k, p, tw, half_step, g) * p.chunk_scale;
        }
      }
    }
    // the G slot sums of a bin sit in adjacent lanes: an xor tree adds them in a fixed order
    for (int o = 1; o < p.G; o <<= 1) {
#pragma unroll
      for (int r = 0; r < ACC; ++r) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
    }
    if (slot == 0) {
      const double scale = p.wscale[0];
#pragma unroll
      for (int r = 0; r < ACC; ++r) {
        const int k = kb + r * kstep;
        if (k >= L) continue;
        if (p.nchunk == 1)
          p.psd[s * L + k] = ((k == 0 || k == p.M) ? acc[r] : 2.0 * acc[r]) * scale;
        else
          p.part[item * L + k] = acc[r];
      }
    }
  }
}

// psd from the chunk sums, added in chunk order
__global__ void __launch_bounds__(256) welch_finish_kernel(const __grid_constant__ WelchParams p) {
  const int L = p.M + 1;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x;
  if (i >= p.nseries * L) return;
  const int64_t s = i / L;
  const int k = static_cast<int>(i % L);
  const double* part = p.part + s * p.nchunk * L + k;
  double acc = part[0] * p.part_scale;
  for (int64_t c = 1; c < p.nchunk; ++c) acc += part[c * L] * p.part_scale;
  p.psd[i] = ((k == 0 || k == p.M) ? acc : 2.0 * acc) * p.wscale[0];
}

}  // namespace b2ins
