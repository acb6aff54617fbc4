// K13: noise identification from an Allan variance curve -- the least-squares fit of IEEE Std 952-1997
// Annex C on the Allan tau grid the curve was computed on (oracle/allan_fit_np.py is the spec).
//
//   model(tau) = C_-2 tau^-2 + C_-1 tau^-1 + C_0 + C_1 tau + C_2 tau^2,   every C_p >= 0,
//   minimise   sum_k w_k (model(tau_k) / v_k - 1)^2,   w_k = floor(n / m_k) - 1,
//
// over the bins with v_k > 0.  The columns a_kp = sqrt(w_k) tau_k^p / v_k are scaled to unit norm once.  The
// non-negative optimum is the feasible support of smallest objective among the 31 non-empty supports of the five
// terms (bit i: the term tau^(i-2)) and the empty one: each support's unconstrained solution comes from a QR
// factorisation of its columns (modified Gram-Schmidt, applied twice, so Q is orthonormal to rounding), and the
// support is feasible when every coefficient on it is > 0.  Supports are visited with fewer terms first, then by
// bitmask; a later one replaces the best only if its objective is lower by more than
// kFitTie * sum_k w_k, so ties go to fewer terms, then to the lower bitmask.  A support with more columns than
// usable bins, or whose R has a diagonal entry <= kFitRank * max |diag|, is skipped.
//
// One warp per series, lane l holds bins l, l + 32, l + 64, l + 96 (the grid has at most 128 bins).  Every sum
// is the lane's own bins in index order, then an xor butterfly: IEEE addition commutes, so every lane ends with
// the same bits and every branch is warp-uniform.  Nothing depends on the series' position, the batch or the
// grid: a series gives the same bits wherever it is fitted.
//
// Outputs per series: Q = sqrt(C_-2 / 3), N = sqrt(C_-1), B = sqrt(C_0) sqrt(pi / (2 ln 2)), K = sqrt(3 C_1),
// R = sqrt(2 C_2), B_min = sqrt(min_k v_k) sqrt(pi / (2 ln 2)).  A NaN, +-inf or negative v_k, or an empty grid,
// gives six NaNs; a zero bin is left out of the fit but counts for B_min; all-zero bins give six zeros.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace b2ins {

constexpr int kFitMaxBins = 128;                 // the Allan grid's cap (b2ins_allan_num_tau)
constexpr int kFitLaneBins = kFitMaxBins / 32;
constexpr int kFitTerms = 5;
constexpr int kFitWarps = 4;                     // series per CTA
constexpr double kFitTie = 1e-12;
constexpr double kFitRank = 1e-13;
constexpr double kFitHuge = 1.7976931348623157e308;   // the largest finite double

struct AllanFitParams {
  const double* var;        // v of series s, bin k at var[s * series_stride + k * bin_stride]
  double* out;              // [nseries][6]
  int64_t nseries;
  int64_t series_stride;
  int64_t bin_stride;
  int ntau;
  double b_scale;           // sqrt(pi / (2 ln 2))
  double nan;               // quiet NaN, from the host: a __longlong_as_double here changes how the
                            // compiler inlines it into K7, whose SASS stays as it was
  double tau[kFitMaxBins];  // m_k * (1 / fs)
  double w[kFitMaxBins];    // floor(n / m_k) - 1
};

__device__ __forceinline__ double fit_warp_sum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// sum over the warp of the lanes' dot products of two bin vectors
__device__ __forceinline__ double fit_dot(const double (&a)[kFitLaneBins], const double (&b)[kFitLaneBins]) {
  double s = a[0] * b[0];
#pragma unroll
  for (int j = 1; j < kFitLaneBins; ++j) s += a[j] * b[j];
  return fit_warp_sum(s);
}

__global__ void __launch_bounds__(kFitWarps * 32) allan_fit_kernel(const AllanFitParams p) {
  const int lane = threadIdx.x & 31;
  const int64_t s = static_cast<int64_t>(blockIdx.x) * kFitWarps + (threadIdx.x >> 5);
  if (s >= p.nseries) return;                       // the whole warp
  double* out = p.out + s * 6;

  double v[kFitLaneBins];
  bool bad = p.ntau == 0;
  double vmin = kFitHuge;
#pragma unroll
  for (int j = 0; j < kFitLaneBins; ++j) {
    const int k = lane + 32 * j;
    v[j] = 0.0;
    if (k < p.ntau) {
      v[j] = p.var[s * p.series_stride + k * p.bin_stride];
      bad |= !(v[j] >= 0.0 && v[j] <= kFitHuge);     // NaN, +-inf or negative
      vmin = v[j] < vmin ? v[j] : vmin;
    }
  }
  if (__any_sync(0xffffffffu, bad)) {
    if (lane < 6) out[lane] = p.nan;
    return;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double other = __shfl_xor_sync(0xffffffffu, vmin, o);
    vmin = other < vmin ? other : vmin;
  }

  // the weighted rows of the usable bins (zeros elsewhere), the column norms, the unit columns d
  double d[kFitTerms][kFitLaneBins], b[kFitLaneBins];
  double wsum = 0.0;
  int usable = 0;
#pragma unroll
  for (int j = 0; j < kFitLaneBins; ++j) {
    const int k = lane + 32 * j;
    const bool use = k < p.ntau && v[j] > 0.0;
    usable += __popc(__ballot_sync(0xffffffffu, use));
    const double t = use ? p.tau[k] : 1.0;
    const double sw = use ? sqrt(p.w[k]) : 0.0;
    const double g = use ? sw / v[j] : 0.0;
    wsum += use ? p.w[k] : 0.0;
    b[j] = sw;
    d[0][j] = g / (t * t);
    d[1][j] = g / t;
    d[2][j] = g;
    d[3][j] = g * t;
    d[4][j] = g * (t * t);
  }
  wsum = fit_warp_sum(wsum);
  double nrm[kFitTerms];
#pragma unroll
  for (int q = 0; q < kFitTerms; ++q) {
    nrm[q] = sqrt(fit_dot(d[q], d[q]));
    const double inv = usable > 0 ? 1.0 / nrm[q] : 0.0;
#pragma unroll
    for (int j = 0; j < kFitLaneBins; ++j) d[q][j] *= inv;
  }

  double best_y[kFitTerms] = {0.0, 0.0, 0.0, 0.0, 0.0};
  double best_obj = wsum;                          // the empty support
  const double tie = kFitTie * wsum;
  for (unsigned visit = 0; visit < kFitTerms * 31; ++visit) {   // fewer terms first, then the lower bitmask
    const unsigned mask = visit % 31 + 1;
    if (__popc(mask) != static_cast<int>(visit / 31) + 1 || __popc(mask) > usable) continue;
    double qc[kFitTerms][kFitLaneBins];            // Q's columns, by term
    double r[kFitTerms][kFitTerms];                // R, upper triangle, by term
    double dmax = 0.0;
#pragma unroll
    for (int c = 0; c < kFitTerms; ++c) {
      if (!(mask >> c & 1u)) continue;
      double x[kFitLaneBins];
#pragma unroll
      for (int j = 0; j < kFitLaneBins; ++j) x[j] = d[c][j];
#pragma unroll
      for (int i = 0; i < c; ++i) r[i][c] = 0.0;
#pragma unroll
      for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
        for (int i = 0; i < c; ++i) {
          if (!(mask >> i & 1u)) continue;
          const double h = fit_dot(qc[i], x);
#pragma unroll
          for (int j = 0; j < kFitLaneBins; ++j) x[j] -= h * qc[i][j];
          r[i][c] += h;
        }
      }
      r[c][c] = sqrt(fit_dot(x, x));
      dmax = r[c][c] > dmax ? r[c][c] : dmax;
      const double inv = 1.0 / r[c][c];
#pragma unroll
      for (int j = 0; j < kFitLaneBins; ++j) qc[c][j] = x[j] * inv;
    }
    bool ok = true;
#pragma unroll
    for (int c = 0; c < kFitTerms; ++c)
      if (mask >> c & 1u) ok = ok && r[c][c] > kFitRank * dmax;    // false for NaN too
    if (!ok) continue;
    double y[kFitTerms];
#pragma unroll
    for (int c = kFitTerms - 1; c >= 0; --c) {
      y[c] = 0.0;
      if (!(mask >> c & 1u)) continue;
      double acc = fit_dot(qc[c], b);
#pragma unroll
      for (int i = c + 1; i < kFitTerms; ++i)
        if (mask >> i & 1u) acc -= r[c][i] * y[i];
      y[c] = acc / r[c][c];
      ok = ok && y[c] > 0.0;
    }
    if (!ok) continue;
    double rr = 0.0;
#pragma unroll
    for (int j = 0; j < kFitLaneBins; ++j) {
      double e = -b[j];
#pragma unroll
      for (int c = 0; c < kFitTerms; ++c) e += d[c][j] * y[c];
      rr += e * e;
    }
    const double obj = fit_warp_sum(rr);
    if (obj < best_obj - tie) {
      best_obj = obj;
#pragma unroll
      for (int c = 0; c < kFitTerms; ++c) best_y[c] = y[c];
    }
  }

  double C[kFitTerms];
#pragma unroll
  for (int c = 0; c < kFitTerms; ++c) C[c] = best_y[c] != 0.0 ? best_y[c] / nrm[c] : 0.0;
  if (lane < 6) {
    double o = sqrt(vmin) * p.b_scale;
    if (lane == 0) o = sqrt(C[0] / 3.0);
    if (lane == 1) o = sqrt(C[1]);
    if (lane == 2) o = sqrt(C[2]) * p.b_scale;
    if (lane == 3) o = sqrt(3.0 * C[3]);
    if (lane == 4) o = sqrt(2.0 * C[4]);
    out[lane] = o;
  }
}

}  // namespace b2ins
