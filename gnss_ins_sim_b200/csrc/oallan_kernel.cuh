// K4o: overlapping Allan variance (NIST SP 1065 eq. 10) on the cluster sizes of K4's grid
// (m = j*10^d, j = 1..9, m <= n/9):
//   S(k, m) = sum_{i=k}^{k+m-1} x_i,   M = n - 2m + 1,
//   avar_o(m) = 1 / (2 m^2 M) * sum_{k=0}^{M-1} (S(k+m, m) - S(k, m))^2.
//
// Every start offset k counts, so the series cannot be cut into clusters as K4 does.  With the
// prefix C[i] = sum_{q<i} (x_q - x_0) a term is the second difference C[k+2m] - 2 C[k+m] + C[k].
//
// Precision.  C grows with the series (accelerometer z at 14.4 M samples: ~1.4e8, one ulp 3e-8,
// against m = 1 differences of 1e-2; a ramp grows it quadratically, and the shift by x_0 does not
// remove a ramp), so C is kept as a double-double (hi, lo) accumulated by TwoSum.  The shift v - x_0 itself
// rounds where the result needs more than 53 bits (an outlier x_0, a wide drift); a double-double add then
// errs by O(u^2) of its operands, not zero.  A term
// is formed from D_L = C[k+L] - C[k] (TwoDiff of the hi parts, exact, plus the lo difference), then
// d = (D_2m.hi - 2 D_m.hi) + (D_2m.lo - 2 D_m.lo): both hi terms are ~2 S and the subtraction is
// exact whenever they are within a factor of two.
//
// Hadamard form (HAD = true in passes 4 and 5): the overlapping Hadamard variance (NIST SP 1065) on the
// same grid, a second difference of three adjacent window sums, so a linear drift cancels exactly:
//   H = n - 3m + 1,
//   hvar(m) = 1 / (6 m^2 H) * sum_{k=0}^{H-1} (S(k+2m, m) - 2 S(k+m, m) + S(k, m))^2
//           = 1 / (6 m^2 H) * sum_{k=0}^{H-1} (C[k+3m] - 3 C[k+2m] + 3 C[k+m] - C[k])^2.
// Precision of its term.  3 h is not exact as 2 h is, so the term is never formed from 3 C or 3 D.  The
// window sums S_i = C[k+(i+1)m] - C[k+im] (i = 0, 1, 2) are taken straight from the prefix, each by an
// exact TwoDiff of the hi parts (its error goes to lo) plus the lo difference; then
//   t = ((S2.hi - S1.hi) - (S1.hi - S0.hi)) + ((S2.lo - S1.lo) - (S1.lo - S0.lo)).
// A hi subtraction is exact (Sterbenz) when its operands are within a factor of two: adjacent window
// sums are whenever a level or a drift dominates them, and the two first differences are whenever the
// drift dominates the term, the cases in which the prefix is large beside the term.  An inexact one
// rounds by at most half an ulp of a first difference of window sums, never of the prefix.  Only the
// lo sums and the final add round otherwise; the lo parts are of the order of an ulp of C.
//
// Passes (one stream, five launches; tiles are fixed by n alone):
//   1 oallan_tile_kernel<false>  per (series, scan tile): the tile's double-double total of x - x_0,
//                                its +inf / -inf counts and NaN / inf flags
//   2 oallan_carry_kernel        per series, sequential over its tiles: the series' class (finite,
//                                inf without NaN, NaN) and the exclusive carry of every tile
//   3 oallan_tile_kernel<true>   per (series, scan tile): C written to the workspace [nseries][n+1]
//   4 oallan_sq_kernel<HAD>      per (series, decade, output tile): the nine sizes j*10^d share the
//                                14 lags {1..10, 12, 14, 16, 18}*10^d of C[k] (Hadamard: 18 lags
//                                {1..10, 12, 14, 15, 16, 18, 21, 24, 27}*10^d); nine partial sums
//   5 oallan_final_kernel<HAD>   per (series, tau): the tiles' partials, folded in a fixed order
//
// Determinism: every sum runs in an order fixed by n (thread-serial runs, fixed butterflies, warps
// and tiles in index order), never by the grid, the batch or the position of a series in it.
//
// Non-finite series.  A prefix difference turns an inf into inf - inf in windows that do not hold
// it, so such series take an exact form instead.  A NaN sample makes every tau NaN.  With +-inf
// (and no NaN) the definitional sum is +inf or NaN: every sample lies in some term's windows, a
// term is inf or NaN when its windows hold an inf, and it is NaN exactly when one window holds both
// signs or both windows hold the same sign.  For these series pass 3 writes the prefix COUNTS of
// +inf (hi) and -inf (lo) samples instead (exact small integers), pass 4 counts the NaN terms with
// the same lags, and pass 5 gives NaN if there is one, else +inf.  A Hadamard term is NaN exactly when
// its signed contributions +S2, -2 S1, +S0 hold both infinities: a window holds both signs, or S2 and
// S0 are infinite with opposite signs, or S1 is infinite with the sign of S2 or of S0.  That is what
// the definitional sum gives in IEEE arithmetic, whatever the order of its additions.  A series of finite
// samples never gives NaN: if its shifted prefix overflows (x_0 = -1e305, the rest +1e305), TwoSum of the
// infinite sum is NaN, and pass 5 reports that series' taus as +inf, which its terms' squares are.
#pragma once
#include <cmath>
#include <cstring>

#include "common.cuh"

namespace b2ins {

constexpr int kOallanScanThreads = 256;
constexpr int kOallanScanPer = 9;                                           // samples per thread
constexpr int kOallanScanTile = kOallanScanThreads * kOallanScanPer;        // 2304
constexpr int kOallanSqThreads = 256;
constexpr int kOallanSqPer = 8;                                             // offsets k per thread
constexpr int kOallanSqTile = kOallanSqThreads * kOallanSqPer;              // 2048
constexpr int kOallanMaxDec = 10;
constexpr int kOallanLags = 14;
constexpr int kOhadLags = 18;

enum { kOallanFinite = 0, kOallanInf = 1, kOallanNan = 2 };

struct OallanParams {
  int64_t n, nseries;
  const double* x;                       // series s, sample t: x[s / inner * outer_stride + s % inner + t * sample_stride]
  int64_t inner, outer_stride, sample_stride;
  int64_t tiles;                         // scan tiles per series: ceil(n / kOallanScanTile)
  double2* c;                            // [nseries][n + 1]: C (finite) or (+inf count, -inf count)
  double2* tot;                          // [nseries][tiles] double-double tile totals
  double2* cnt;                          // [nseries][tiles] (+inf, -inf) counts of the tile
  double2* carry;                        // [nseries][tiles] exclusive carry, in the series' form
  int* tflag;                            // [nseries][tiles] bit 0: an inf, bit 1: a NaN
  int* sflag;                            // [nseries] kOallanFinite / Inf / Nan
  // pass 4
  int ndec;
  int64_t sq_tiles;                      // output tiles per (series, decade): ceil(n / kOallanSqTile)
  int jmax[kOallanMaxDec];
  int64_t p10[kOallanMaxDec];
  double* partial;                       // [nseries][ndec][sq_tiles][9]
};

// ---- double-double arithmetic (error-free transformations; no FMA contraction) ------------------
struct DD {
  double hi, lo;
};

__device__ __forceinline__ DD two_sum(double a, double b) {
  const double s = __dadd_rn(a, b);
  const double bb = __dsub_rn(s, a);
  const double e = __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb));
  return {s, e};
}

__device__ __forceinline__ DD quick_two_sum(double a, double b) {
  const double s = __dadd_rn(a, b);
  return {s, __dsub_rn(b, __dsub_rn(s, a))};
}

__device__ __forceinline__ DD dd_add_d(DD a, double b) {
  const DD s = two_sum(a.hi, b);
  return quick_two_sum(s.hi, __dadd_rn(s.lo, a.lo));
}

__device__ __forceinline__ DD dd_add(DD a, DD b) {
  const DD s = two_sum(a.hi, b.hi);
  return quick_two_sum(s.hi, __dadd_rn(s.lo, __dadd_rn(a.lo, b.lo)));
}

// a - b for two prefix values: exact TwoDiff of the hi parts, the lo parts added to its error
__device__ __forceinline__ DD dd_diff(double2 a, double2 b) {
  const DD s = two_sum(a.x, -b.x);
  return {s.hi, __dadd_rn(s.lo, __dsub_rn(a.y, b.y))};
}

// the element combine of the scan: double-double for finite series, plain (exact) count addition
// for the +inf / -inf counts
template <bool COUNT>
__device__ __forceinline__ DD scan_op(DD a, DD b) {
  if (COUNT) return {a.hi + b.hi, a.lo + b.lo};
  return dd_add(a, b);
}

__device__ __forceinline__ const double* oallan_base(const OallanParams& p, int64_t s) {
  return p.x + (s / p.inner) * p.outer_stride + (s % p.inner);
}

// Block-wide inclusive scan of one value per thread (Hillis-Steele in shared memory, fixed order).
template <bool COUNT>
__device__ __forceinline__ DD block_scan(DD v, DD* sh) {
  const int tid = threadIdx.x;
  sh[tid] = v;
  __syncthreads();
  for (int o = 1; o < kOallanScanThreads; o <<= 1) {
    const DD u = (tid >= o) ? sh[tid - o] : DD{0.0, 0.0};
    __syncthreads();
    if (tid >= o) {
      v = scan_op<COUNT>(u, v);
      sh[tid] = v;
    }
    __syncthreads();
  }
  return v;
}

// Pass 3 for one tile: thread t scans samples 9t .. 9t+8 serially (loc), the thread totals are
// scanned across the block, and C = carry + (threads before) + loc.  COUNT: the +inf / -inf counts.
template <bool COUNT>
__device__ __forceinline__ void oallan_tile_write(const OallanParams& p, int64_t s, int64_t t, const double* raw,
                                                  int cnt, double x0, DD* sh) {
  const int tid = threadIdx.x, b0 = tid * kOallanScanPer;
  DD loc[kOallanScanPer];
  DD run{0.0, 0.0};
#pragma unroll
  for (int q = 0; q < kOallanScanPer; ++q) {
    const double v = raw[b0 + q];
    const bool in = b0 + q < cnt;
    if (COUNT)
      run = {run.hi + ((in && v == INFINITY) ? 1.0 : 0.0), run.lo + ((in && v == -INFINITY) ? 1.0 : 0.0)};
    else if (in)
      run = dd_add_d(run, v - x0);
    loc[q] = run;
  }
  block_scan<COUNT>(run, sh);   // sh[i]: inclusive total of threads 0..i
  const double2 cr = p.carry[s * p.tiles + t];
  DD ex{cr.x, cr.y};
  if (tid > 0) ex = scan_op<COUNT>(ex, sh[tid - 1]);
  double2* out = p.c + s * (p.n + 1) + t * kOallanScanTile + 1;
#pragma unroll
  for (int q = 0; q < kOallanScanPer; ++q) {
    if (b0 + q < cnt) {
      const DD c = scan_op<COUNT>(ex, loc[q]);
      out[b0 + q] = make_double2(c.hi, c.lo);
    }
  }
  if (t == 0 && tid == 0) p.c[s * (p.n + 1)] = make_double2(0.0, 0.0);
}

// Passes 1 and 3: one CTA per (series, scan tile), the tile staged in shared memory by coalesced
// loads.  WRITE = false: the tile's totals and flags; WRITE = true: C.
template <bool WRITE>
__global__ void __launch_bounds__(kOallanScanThreads) oallan_tile_kernel(const __grid_constant__ OallanParams p) {
  __shared__ double raw[kOallanScanTile];
  __shared__ DD sh[kOallanScanThreads];
  __shared__ int sh_flag;
  const int64_t s = blockIdx.x / p.tiles;
  const int64_t t = blockIdx.x % p.tiles;
  const int tid = threadIdx.x;
  const int mode = WRITE ? p.sflag[s] : kOallanFinite;
  if (WRITE && mode == kOallanNan) return;   // pass 5 writes NaN; C is not needed
  const double* base = oallan_base(p, s);
  const int64_t t0 = t * kOallanScanTile;
  const int cnt = static_cast<int>(min64(kOallanScanTile, p.n - t0));
  const double x0 = base[0];
  {
    double v[kOallanScanPer];   // every load is issued before the first store
#pragma unroll
    for (int q = 0; q < kOallanScanPer; ++q) {
      const int i = tid + q * kOallanScanThreads;
      v[q] = (i < cnt) ? base[(t0 + i) * p.sample_stride] : 0.0;
    }
#pragma unroll
    for (int q = 0; q < kOallanScanPer; ++q) raw[tid + q * kOallanScanThreads] = v[q];
  }
  if (!WRITE && tid == 0) sh_flag = 0;
  __syncthreads();
  if (WRITE) {
    if (mode == kOallanInf)
      oallan_tile_write<true>(p, s, t, raw, cnt, x0, sh);
    else
      oallan_tile_write<false>(p, s, t, raw, cnt, x0, sh);
    return;
  }
  const int b0 = tid * kOallanScanPer;
  DD run{0.0, 0.0}, pn{0.0, 0.0};   // pn: (+inf, -inf) counts
  int flag = 0;
#pragma unroll
  for (int q = 0; q < kOallanScanPer; ++q) {
    const double v = raw[b0 + q];
    if (b0 + q < cnt) {
      run = dd_add_d(run, v - x0);
      if (isnan(v)) flag |= 2;
      if (isinf(v)) {
        flag |= 1;
        if (v > 0.0) pn.hi += 1.0; else pn.lo += 1.0;
      }
    }
  }
  if (flag) atomicOr(&sh_flag, flag);
  block_scan<false>(run, sh);
  const DD total = sh[kOallanScanThreads - 1];
  __syncthreads();
  block_scan<true>(pn, sh);
  if (tid == 0) {
    p.tot[s * p.tiles + t] = make_double2(total.hi, total.lo);
    p.cnt[s * p.tiles + t] = make_double2(sh[kOallanScanThreads - 1].hi, sh[kOallanScanThreads - 1].lo);
    p.tflag[s * p.tiles + t] = sh_flag;
  }
}

// Pass 2: one thread per series walks its tiles in order.
__global__ void __launch_bounds__(128) oallan_carry_kernel(const __grid_constant__ OallanParams p) {
  const int64_t s = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (s >= p.nseries) return;
  int f = 0;
  for (int64_t t = 0; t < p.tiles; ++t) f |= p.tflag[s * p.tiles + t];
  const int mode = (f & 2) ? kOallanNan : (f & 1) ? kOallanInf : kOallanFinite;
  p.sflag[s] = mode;
  if (mode == kOallanNan) return;
  const double2* src = (mode == kOallanInf ? p.cnt : p.tot) + s * p.tiles;
  double2* dst = p.carry + s * p.tiles;
  DD run{0.0, 0.0};
  constexpr int kAhead = 8;   // loads issued ahead of the dependent adds
  for (int64_t t0 = 0; t0 < p.tiles; t0 += kAhead) {
    double2 v[kAhead];
#pragma unroll
    for (int q = 0; q < kAhead; ++q) v[q] = (t0 + q < p.tiles) ? src[t0 + q] : make_double2(0.0, 0.0);
#pragma unroll
    for (int q = 0; q < kAhead; ++q) {
      if (t0 + q < p.tiles) {
        dst[t0 + q] = make_double2(run.hi, run.lo);
        run = (mode == kOallanInf) ? scan_op<true>(run, {v[q].x, v[q].y}) : dd_add(run, {v[q].x, v[q].y});
      }
    }
  }
}

// Pass 4.  Thread tid takes offsets k = k0 + tid + 256 q; for each it loads the prefix at the lags
// once.  Allan: the 14 lag differences D_L = C[k + L 10^d] - C[k], and the nine terms from them (size
// j: D_j and D_2j).  Hadamard: the 18 lags, and size j's window sums between lags 0, j, 2j and 3j.
template <bool HAD>
__global__ void __launch_bounds__(kOallanSqThreads) oallan_sq_kernel(const __grid_constant__ OallanParams p) {
  constexpr int kSpan = HAD ? 3 : 2;          // windows per term
  constexpr int kLags = HAD ? kOhadLags : kOallanLags;
  __shared__ double red[kOallanSqThreads / 32][9];
  const int64_t per_series = static_cast<int64_t>(p.ndec) * p.sq_tiles;
  const int64_t s = blockIdx.x / per_series;
  const int64_t r = blockIdx.x % per_series;
  const int d = static_cast<int>(r / p.sq_tiles);
  const int64_t tile = r % p.sq_tiles;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int mode = p.sflag[s];
  const int jmax = p.jmax[d];
  const int64_t u = p.p10[d];
  const int64_t n = p.n;
  const double2* c = p.c + s * (n + 1);
  double acc[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) acc[j] = 0.0;
  constexpr int kLag[kOallanLags] = {1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 16, 18};
  constexpr int kHadLag[kOhadLags] = {1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 15, 16, 18, 21, 24, 27};
  constexpr int kHad2[9] = {1, 3, 5, 7, 9, 10, 11, 13, 14};       // slot of lag 2j in kHadLag
  constexpr int kHad3[9] = {2, 5, 8, 10, 12, 14, 15, 16, 17};     // slot of lag 3j
  if (mode != kOallanNan) {
    for (int q = 0; q < kOallanSqPer; ++q) {
      const int64_t k = tile * kOallanSqTile + q * kOallanSqThreads + tid;
      if (k + kSpan * u > n) break;   // no term of any size of this decade starts here
      const double2 c0 = __ldg(c + k);
      double2 cl[kLags];
#pragma unroll
      for (int l = 0; l < kLags; ++l) {
        const int64_t i = k + (HAD ? kHadLag[l] : kLag[l]) * u;
        cl[l] = (i <= n) ? __ldg(c + i) : c0;
      }
#pragma unroll
      for (int j = 1; j <= 9; ++j) {
        if (HAD) {
          if (j <= jmax && k + 3 * j * u <= n) {
            const double2 c1 = cl[j - 1], c2 = cl[kHad2[j - 1]], c3 = cl[kHad3[j - 1]];
            if (mode == kOallanFinite) {   // window sums S0, S1, S2 (see the file comment)
              const DD s0 = dd_diff(c1, c0), s1 = dd_diff(c2, c1), s2 = dd_diff(c3, c2);
              const double t = __dadd_rn(__dsub_rn(__dsub_rn(s2.hi, s1.hi), __dsub_rn(s1.hi, s0.hi)),
                                         __dsub_rn(__dsub_rn(s2.lo, s1.lo), __dsub_rn(s1.lo, s0.lo)));
              acc[j - 1] = fma(t, t, acc[j - 1]);
            } else {   // +inf (x) / -inf (y) counts; an inf of S1 enters the term with its sign flipped
              const bool pos = c1.x > c0.x || c2.y > c1.y || c3.x > c2.x;
              const bool neg = c1.y > c0.y || c2.x > c1.x || c3.y > c2.y;
              acc[j - 1] += (pos && neg) ? 1.0 : 0.0;
            }
          }
          continue;
        }
        if (j <= jmax && k + 2 * j * u <= n) {
          const int l1 = j - 1, l2 = (j <= 5) ? 2 * j - 1 : j + 4;   // lags j and 2j
          const DD a = dd_diff(cl[l1], c0), b = dd_diff(cl[l2], c0);
          if (mode == kOallanFinite) {
            const double t = __dadd_rn(__dsub_rn(b.hi, 2.0 * a.hi), __dsub_rn(b.lo, 2.0 * a.lo));
            acc[j - 1] = fma(t, t, acc[j - 1]);
          } else {   // counts of +inf (hi) and -inf (lo) in the first window [k, k+m) and the second
            const double pa = a.hi, na = a.lo, pb = b.hi - a.hi, nb = b.lo - a.lo;
            const bool nan_term = (pa > 0.0 && na > 0.0) || (pb > 0.0 && nb > 0.0) ||
                                  (pa > 0.0 && pb > 0.0) || (na > 0.0 && nb > 0.0);
            acc[j - 1] += nan_term ? 1.0 : 0.0;
          }
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    double v = acc[j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][j] = v;
  }
  __syncthreads();
  if (tid < 9) {
    double v = 0.0;
    for (int w = 0; w < kOallanSqThreads / 32; ++w) v += red[w][tid];
    p.partial[((s * p.ndec + d) * p.sq_tiles + tile) * 9 + tid] = v;
  }
}

struct OallanFinalParams {
  int64_t n, nseries, sq_tiles;
  int ntau, ndec;
  double ts;
  const double* partial;
  const int* sflag;
  double* avar;   // [nseries][ntau]
  double* tau;    // [ntau]
  int64_t m[128];
  int dec_of[128];
  int j_of[128];
};

// Pass 5: one warp per (series, tau), lanes over the tiles in order, then a fixed butterfly.
template <bool HAD>
__global__ void __launch_bounds__(128) oallan_final_kernel(const __grid_constant__ OallanFinalParams p) {
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (idx >= p.nseries * p.ntau) return;
  const int lane = threadIdx.x & 31;
  const int64_t s = idx / p.ntau;
  const int i = static_cast<int>(idx % p.ntau);
  const double* part = p.partial + ((s * p.ndec + p.dec_of[i]) * p.sq_tiles) * 9 + (p.j_of[i] - 1);
  double v = 0.0;
  for (int64_t t = lane; t < p.sq_tiles; t += 32) v += part[t * 9];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) {
    const double m = static_cast<double>(p.m[i]);
    const int mode = p.sflag[s];
    double a;
    if (mode == kOallanNan)
      a = NAN;
    else if (mode == kOallanInf)
      a = v > 0.0 ? NAN : INFINITY;
    else if (isnan(v))   // finite samples: only an overflowing prefix (inf - inf in its TwoSum) gives NaN
      a = INFINITY;
    else if (HAD)
      a = v / (6.0 * m * m * static_cast<double>(p.n - 3 * p.m[i] + 1));
    else
      a = v / (2.0 * m * m * static_cast<double>(p.n - 2 * p.m[i] + 1));
    p.avar[s * p.ntau + i] = a;
    if (s == 0) p.tau[i] = m * p.ts;
  }
}

// decades d with 10^d <= floor(n / 9): the decades of K4's tau grid
inline int oallan_decades(int64_t n) {
  const int64_t max_bin = n / 9;
  int nd = 0;
  for (int64_t u = 1; nd < kOallanMaxDec && u <= max_bin; u *= 10) ++nd;
  return nd;
}

struct OallanLayout {
  int64_t c, tot, cnt, carry, tflag, sflag, partial, bytes;   // byte offsets into the workspace
};

inline OallanLayout oallan_layout(int64_t n, int64_t nseries) {
  auto up = [](int64_t b) { return (b + 255) & ~int64_t(255); };
  const int64_t tiles = (n + kOallanScanTile - 1) / kOallanScanTile;
  const int64_t sq_tiles = (n + kOallanSqTile - 1) / kOallanSqTile;
  OallanLayout l;
  l.c = 0;
  l.tot = up(l.c + nseries * (n + 1) * 16);
  l.cnt = up(l.tot + nseries * tiles * 16);
  l.carry = up(l.cnt + nseries * tiles * 16);
  l.tflag = up(l.carry + nseries * tiles * 16);
  l.sflag = up(l.tflag + nseries * tiles * 4);
  l.partial = up(l.sflag + nseries * 4);
  l.bytes = up(l.partial + nseries * oallan_decades(n) * sq_tiles * 9 * 8);
  return l;
}

inline int64_t oallan_workspace_bytes(int64_t n, int64_t nseries) {
  if (n <= 0 || nseries <= 0) return 16;
  return oallan_layout(n, nseries).bytes + 256;   // + 256: the caller's base need not be aligned
}

// returns 0 on success; mult/ntau: the tau grid (b2ins_allan_num_tau); hadamard: the Hadamard form of
// passes 4 and 5 (avar is then hvar)
inline int oallan_launch(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner,
                         int64_t outer_stride, int64_t sample_stride, const int64_t* mult, int ntau,
                         double* avar, double* tau, void* workspace, cudaStream_t st, bool hadamard) {
  OallanParams p;
  std::memset(&p, 0, sizeof(p));
  OallanFinalParams fp;
  std::memset(&fp, 0, sizeof(fp));
  p.n = n;
  p.nseries = nseries;
  p.x = x;
  p.inner = inner;
  p.outer_stride = outer_stride;
  p.sample_stride = sample_stride;
  p.tiles = (n + kOallanScanTile - 1) / kOallanScanTile;
  p.ndec = oallan_decades(n);
  p.sq_tiles = (n + kOallanSqTile - 1) / kOallanSqTile;
  {
    int64_t u = 1;
    for (int d = 0; d < p.ndec; ++d, u *= 10) p.p10[d] = u;
    for (int i = 0; i < ntau; ++i) {
      int d = 0;
      while (d < p.ndec && !(mult[i] % p.p10[d] == 0 && mult[i] / p.p10[d] >= 1 && mult[i] / p.p10[d] <= 9)) ++d;
      if (d == p.ndec) return 1;
      const int j = static_cast<int>(mult[i] / p.p10[d]);
      if (j > p.jmax[d]) p.jmax[d] = j;
      fp.m[i] = mult[i];
      fp.dec_of[i] = d;
      fp.j_of[i] = j;
    }
  }
  if (nseries * p.tiles >= (int64_t(1) << 31) || nseries * p.ndec * p.sq_tiles >= (int64_t(1) << 31)) return 4;
  const OallanLayout l = oallan_layout(n, nseries);
  char* ws = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(workspace) + 255) & ~uintptr_t(255));
  p.c = reinterpret_cast<double2*>(ws + l.c);
  p.tot = reinterpret_cast<double2*>(ws + l.tot);
  p.cnt = reinterpret_cast<double2*>(ws + l.cnt);
  p.carry = reinterpret_cast<double2*>(ws + l.carry);
  p.tflag = reinterpret_cast<int*>(ws + l.tflag);
  p.sflag = reinterpret_cast<int*>(ws + l.sflag);
  p.partial = reinterpret_cast<double*>(ws + l.partial);
  const unsigned scan_grid = static_cast<unsigned>(nseries * p.tiles);
  oallan_tile_kernel<false><<<scan_grid, kOallanScanThreads, 0, st>>>(p);
  oallan_carry_kernel<<<static_cast<unsigned>((nseries + 127) / 128), 128, 0, st>>>(p);
  oallan_tile_kernel<true><<<scan_grid, kOallanScanThreads, 0, st>>>(p);
  const unsigned sq_grid = static_cast<unsigned>(nseries * p.ndec * p.sq_tiles);
  if (hadamard)
    oallan_sq_kernel<true><<<sq_grid, kOallanSqThreads, 0, st>>>(p);
  else
    oallan_sq_kernel<false><<<sq_grid, kOallanSqThreads, 0, st>>>(p);
  fp.n = n;
  fp.nseries = nseries;
  fp.sq_tiles = p.sq_tiles;
  fp.ntau = ntau;
  fp.ndec = p.ndec;
  fp.ts = 1.0 / fs;
  fp.partial = p.partial;
  fp.sflag = p.sflag;
  fp.avar = avar;
  fp.tau = tau;
  const int64_t total = nseries * ntau;
  const unsigned final_grid = static_cast<unsigned>((total + 3) / 4);
  if (hadamard)
    oallan_final_kernel<true><<<final_grid, 128, 0, st>>>(fp);
  else
    oallan_final_kernel<false><<<final_grid, 128, 0, st>>>(fp);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

}  // namespace b2ins
