// K5: vibration time series from a single-sided PSD -- time_series_from_psd
// (gnss_ins_sim/psd/time_series_from_psd.py:17-65), for runs x 3 axes of one sensor.
//
//   N   = n rounded up to even, capped at 16384 (:36-43);  L = N/2 + 1
//   sxx = np.interp(linspace(0, fs/2, L), freq, sxx) unless len(freq) == L (:45-50)
//   sxx[1:L-1] *= 0.5 ; ax = sqrt(sxx N fs) ; phi = pi randn(L) ; xk = ax exp(j phi) (:51-54)
//   x = real(ifft([xk, conj(xk[-2:0:-1])])) (:55-57), tiled to n by the consumer (t % N)
//
// The real part of that inverse DFT is a cosine synthesis,
//   x[m] = (1/N) [ A_0 + (-1)^m A_{L-1} + 2 sum_{k=1}^{L-2} (A_k cos(2 pi k m / N) - B_k sin(2 pi k m / N)) ]
// with A_k + j B_k = ax_k exp(j phi_k).  Kernel 1 draws the phases (Philox normal z0 of
// (t = k, draw = kDrawPsd + 3 sensor + axis, run)) and writes (A_k, B_k); kernel 2 evaluates the
// sum for one output sample per thread, rotating (cos, sin) by 2 pi m / N per k and
// re-seeding it exactly (integer k m mod N, sincospi) every kPsdReseed terms.  N need not be a
// power of two (N = n for short runs): this direct synthesis is the fallback for the lengths the FFT
// path below does not take.
//
// FFT path (psd_fft_kernel).  The Hermitian inverse DFT of length N is one complex inverse DFT of
// length M = N/2:  Z_k = (X_k + conj X_{M-k}) + j (X_k - conj X_{M-k}) e^{2 pi j k / N},
// z = sum_k Z_k e^{2 pi j k m / M},  x[2m] = Re z_m / N,  x[2m+1] = Im z_m / N.  A persistent CTA keeps
// the work array (M or P complex doubles) and a twiddle table in shared memory and runs an in-place
// radix-2 transform per series:
//   * M a power of two (N = 16384 for every run longer than 16383 samples): decimation in time on the
//     bit-reversed placement, natural-order output, coalesced stores;
//   * any other M <= 4096: Bluestein -- the chirp product a_k = Z_k c_k (c_k = e^{j pi k^2 / M}, k^2
//     reduced mod 2M in integers) convolved with conj(c) by two transforms of length P = 2^ceil(log2(2M-1))
//     (the transform of the chirp is made once per launch by psd_chirp_kernel and read from L2).
// O(N log N) instead of O(N L): 16384-sample series go from 8e3 to ~1e6 per second.
#pragma once
#include "common.cuh"

namespace b2ins {

constexpr int kPsdThreads = 256;
constexpr int kPsdReseed = 32;
constexpr int kPsdChunk = 1024;  // (A,B) pairs staged per shared-memory chunk

struct PsdParams {
  double fs;
  int64_t runs, run_offset;
  int N, L, L0, sensor;
  int interp;          // 1: interpolate the table to L points
  uint32_t k0, k1;
  const double* freq;  // [L0]
  const double* sxx;   // [3][L0]
  double* ab;          // workspace [runs][3][L][2]
  double* series;      // [runs][3][N]
};

// np.interp(x, xp, fp): linear, clamped to the end values
__device__ __forceinline__ double interp_clamped(double x, const double* xp, const double* fp, int n) {
  if (x <= xp[0]) return fp[0];
  if (x >= xp[n - 1]) return fp[n - 1];
  int lo = 0, hi = n - 1;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (xp[mid] <= x)
      lo = mid;
    else
      hi = mid;
  }
  const double slope = (fp[hi] - fp[lo]) / (xp[hi] - xp[lo]);
  return slope * (x - xp[lo]) + fp[lo];
}

__global__ void __launch_bounds__(kPsdThreads) psd_phase_kernel(const __grid_constant__ PsdParams p) {
  const int64_t series = blockIdx.y;  // run * 3 + axis
  const int64_t run = series / 3;
  const int axis = static_cast<int>(series % 3);
  const int k = blockIdx.x * kPsdThreads + threadIdx.x;
  if (k >= p.L) return;
  const int64_t grun = p.run_offset + run;
  const double* tab = p.sxx + static_cast<int64_t>(axis) * p.L0;
  double sx;
  if (p.interp) {
    // np.linspace(0, fs/2, L)[k] = k * step, step = (fs/2) / (L - 1) (endpoint exact)
    const double stop = p.fs / 2.0;
    const double fk = (k == p.L - 1) ? stop : k * (stop / static_cast<double>(p.L - 1));
    sx = interp_clamped(fk, p.freq, tab, p.L0);
  } else {
    sx = tab[k];
  }
  if (k >= 1 && k < p.L - 1) sx = 0.5 * sx;
  const double ax = sqrt(sx * static_cast<double>(p.N) * p.fs);
  const Normal2 z = normal_pair(static_cast<uint32_t>(k), kDrawPsd + 3 * p.sensor + axis,
                                static_cast<uint32_t>(grun), static_cast<uint32_t>(grun >> 32), p.k0, p.k1);
  double s, c;
  sincos(kPi * z.z0, &s, &c);  // phi = math.pi * randn
  double* o = p.ab + (series * p.L + k) * 2;
  o[0] = ax * c;
  o[1] = ax * s;
}

__global__ void __launch_bounds__(kPsdThreads) psd_synth_kernel(const __grid_constant__ PsdParams p) {
  __shared__ double sh[kPsdChunk * 2];
  const int64_t series = blockIdx.y;
  const int m = blockIdx.x * kPsdThreads + threadIdx.x;
  const bool live = m < p.N;
  const double* ab = p.ab + series * p.L * 2;
  const int mm = live ? m : 0;
  // rotation by delta = 2 pi m / N
  double sd, cd;
  sincospi(2.0 * static_cast<double>(mm) / static_cast<double>(p.N), &sd, &cd);
  double acc = 0.0;
  double c = 1.0, s = 0.0;
  for (int k0 = 0; k0 < p.L; k0 += kPsdChunk) {
    const int cnt = min(kPsdChunk, p.L - k0);
    __syncthreads();
    for (int i = threadIdx.x; i < cnt * 2; i += kPsdThreads) sh[i] = ab[k0 * 2 + i];
    __syncthreads();
    for (int i = 0; i < cnt; ++i) {
      const int k = k0 + i;
      if ((k % kPsdReseed) == 0) {
        // exact angle: 2 pi ((k m) mod N) / N
        const int64_t r = (static_cast<int64_t>(k) * mm) % p.N;
        sincospi(2.0 * static_cast<double>(r) / static_cast<double>(p.N), &s, &c);
      }
      const double w = (k == 0 || k == p.L - 1) ? 1.0 : 2.0;
      // Re((A + jB)(c + js)) = A c - B s
      acc = fma(w, fma(sh[2 * i], c, -sh[2 * i + 1] * s), acc);
      const double cn = fma(c, cd, -s * sd);
      s = fma(s, cd, c * sd);
      c = cn;
    }
  }
  if (live) p.series[series * p.N + m] = acc / static_cast<double>(p.N);
}

// ---- FFT path -----------------------------------------------------------------------------------
constexpr int kFftThreads = 512;

struct PsdFftParams {
  int64_t nseries;       // runs * 3
  int N, L, M, P, logP;  // P = M (power of two) or the Bluestein length
  int bluestein;
  const double* ab;      // [nseries][L][2] from psd_phase_kernel
  double2* bhat;         // [P] transform of the conjugate chirp (Bluestein)
  double* series;        // [nseries][N]
};

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(fma(a.x, b.x, -a.y * b.y), fma(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ int bitrev(int i, int bits) { return static_cast<int>(__brev(static_cast<unsigned>(i)) >> (32 - bits)); }

// tw[j] = e^{+2 pi j / P}, j < P/2
__device__ __forceinline__ void fft_twiddles(double2* tw, int P) {
  for (int j = threadIdx.x; j < P / 2; j += blockDim.x) {
    double s, c;
    sincospi(2.0 * static_cast<double>(j) / static_cast<double>(P), &s, &c);
    tw[j] = make_double2(c, s);
  }
}
// in-place radix-2, decimation in time: bit-reversed input -> natural output; SIGN = +1: e^{+...}.
// `batch` transforms of length P lie back to back in x: butterfly b of the batch indexes the same
// pair and twiddle as in a single transform, because half divides P / 2.
template <int SIGN>
__device__ __forceinline__ void fft_dit(double2* x, const double2* tw, int P, int batch = 1) {
  for (int half = 1; half < P; half <<= 1) {
    const int tstep = P / (2 * half);
    __syncthreads();
    for (int b = threadIdx.x; b < (P / 2) * batch; b += blockDim.x) {
      const int j = b & (half - 1);
      const int i = ((b - j) << 1) + j;
      double2 w = tw[j * tstep];
      if (SIGN < 0) w.y = -w.y;
      const double2 u = x[i], t = cmul(w, x[i + half]);
      x[i] = make_double2(u.x + t.x, u.y + t.y);
      x[i + half] = make_double2(u.x - t.x, u.y - t.y);
    }
  }
  __syncthreads();
}
// decimation in frequency: natural input -> bit-reversed output
template <int SIGN>
__device__ __forceinline__ void fft_dif(double2* x, const double2* tw, int P, int batch = 1) {
  for (int half = P / 2; half >= 1; half >>= 1) {
    const int tstep = P / (2 * half);
    __syncthreads();
    for (int b = threadIdx.x; b < (P / 2) * batch; b += blockDim.x) {
      const int j = b & (half - 1);
      const int i = ((b - j) << 1) + j;
      double2 w = tw[j * tstep];
      if (SIGN < 0) w.y = -w.y;
      const double2 u = x[i], v = x[i + half];
      x[i] = make_double2(u.x + v.x, u.y + v.y);
      x[i + half] = cmul(w, make_double2(u.x - v.x, u.y - v.y));
    }
  }
  __syncthreads();
}
// c_k = e^{j pi k^2 / M}, the angle reduced exactly: k^2 mod 2M
__device__ __forceinline__ double2 chirp(int k, int M) {
  const int64_t r = (static_cast<int64_t>(k) * k) % (2 * static_cast<int64_t>(M));
  double s, c;
  sincospi(static_cast<double>(r) / static_cast<double>(M), &s, &c);
  return make_double2(c, s);
}
// Z_k of the length-M complex transform that carries the Hermitian length-N one (k < M)
__device__ __forceinline__ double2 packed_bin(const double* ab, int k, int M, int N) {
  if (k == 0)   // the imaginary parts of X_0 and X_M do not reach the real part of the inverse transform
    return make_double2(ab[0] + ab[2 * M], ab[0] - ab[2 * M]);
  const double xr = ab[2 * k], xi = ab[2 * k + 1];
  const double yr = ab[2 * (M - k)], yi = -ab[2 * (M - k) + 1];       // conj X_{M-k}
  double s, c;
  sincospi(2.0 * static_cast<double>(k) / static_cast<double>(N), &s, &c);
  const double2 o = cmul(make_double2(xr - yr, xi - yi), make_double2(c, s));
  return make_double2((xr + yr) - o.y, (xi + yi) + o.x);              // E + j O
}

// transform of the wrapped conjugate chirp, once per launch (one CTA)
__global__ void __launch_bounds__(kFftThreads) psd_chirp_kernel(const __grid_constant__ PsdFftParams p) {
  extern __shared__ __align__(16) unsigned char fft_smem[];
  double2* x = reinterpret_cast<double2*>(fft_smem);
  double2* tw = x + p.P;
  fft_twiddles(tw, p.P);
  for (int i = threadIdx.x; i < p.P; i += blockDim.x) x[i] = make_double2(0.0, 0.0);
  __syncthreads();
  for (int j = threadIdx.x; j < p.M; j += blockDim.x) {
    double2 c = chirp(j, p.M);
    c.y = -c.y;
    x[bitrev(j, p.logP)] = c;
    if (j > 0) x[bitrev(p.P - j, p.logP)] = c;
  }
  fft_dit<-1>(x, tw, p.P);
  for (int i = threadIdx.x; i < p.P; i += blockDim.x) p.bhat[i] = x[i];
}

__global__ void __launch_bounds__(kFftThreads, 1) psd_fft_kernel(const __grid_constant__ PsdFftParams p) {
  extern __shared__ __align__(16) unsigned char fft_smem[];
  double2* x = reinterpret_cast<double2*>(fft_smem);
  double2* tw = x + p.P;
  fft_twiddles(tw, p.P);
  const double inv_n = 1.0 / static_cast<double>(p.N);
  for (int64_t series = blockIdx.x; series < p.nseries; series += gridDim.x) {
    const double* ab = p.ab + series * p.L * 2;
    double* out = p.series + series * p.N;
    __syncthreads();     // the previous series has left the work array
    if (!p.bluestein) {
      for (int k = threadIdx.x; k < p.M; k += blockDim.x) x[bitrev(k, p.logP)] = packed_bin(ab, k, p.M, p.N);
      fft_dit<1>(x, tw, p.P);
      for (int m = threadIdx.x; m < p.M; m += blockDim.x) {
        const double2 z = x[m];
        reinterpret_cast<double2*>(out)[m] = make_double2(z.x * inv_n, z.y * inv_n);
      }
    } else {
      for (int i = threadIdx.x; i < p.P; i += blockDim.x) x[i] = make_double2(0.0, 0.0);
      __syncthreads();
      for (int k = threadIdx.x; k < p.M; k += blockDim.x)
        x[bitrev(k, p.logP)] = cmul(packed_bin(ab, k, p.M, p.N), chirp(k, p.M));
      fft_dit<-1>(x, tw, p.P);                                  // natural order
      for (int i = threadIdx.x; i < p.P; i += blockDim.x) x[i] = cmul(x[i], p.bhat[i]);
      fft_dif<1>(x, tw, p.P);                                   // bit-reversed order, unnormalised
      const double scale = inv_n / static_cast<double>(p.P);
      for (int m = threadIdx.x; m < p.M; m += blockDim.x) {
        const double2 z = cmul(x[bitrev(m, p.logP)], chirp(m, p.M));
        reinterpret_cast<double2*>(out)[m] = make_double2(z.x * scale, z.y * scale);
      }
    }
  }
}

// 0: no FFT path for this length (the direct synthesis takes it); else P, with *bluestein set
inline int psd_fft_plan(int N, int* bluestein) {
  const int M = N / 2;
  if (N % 2 != 0 || M < 8) return 0;
  if ((M & (M - 1)) == 0) {
    *bluestein = 0;
    return M;
  }
  if (M > 4096) return 0;
  int P = 1;
  while (P < 2 * M - 1) P <<= 1;
  *bluestein = 1;
  return P;
}

inline int psd_series_len(int64_t n) {
  int64_t N = n;
  if (n % 2 != 0) N = n + 1;
  if (N > 16384) N = 16384;
  return static_cast<int>(N);
}

}  // namespace b2ins
