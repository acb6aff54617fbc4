// K10: soft- and hard-iron magnetometer calibration (MagCalibrate, MagCalibration.c:34-306, behind
// demo_algorithms/mag_calibrate.py) for every run at once.  One CTA per run, nothing materialised:
//   pass 1  per segment, the moments of d = m - t (t = the run's first x-segment row): sum d [3], sum d d^T [6]
//           and the ten cubic monomials sum d_i d_j d_k [10];
//   the plane-fit normals (M^T M) v = M^T 1 from the moments shifted back: the rows of O;
//   pass 2  per segment, max and min of the two columns of c = O m whose ranges give the sensitivities;
//   the sphere fit [2u, 1] p' = |u|^2 on u = S d, S = diag(s) O, as a linear transform of the pass-1 moments,
//           then hard_iron = [p' + S t, sqrt(p'_3 + |p'|^2)].  The 4x4 system is equilibrated by a power of two
//           (u -> f u, f ~ 1 / rms |u|), so its pivot rule does not depend on the units of the samples and
//           the result scales with them bit for bit wherever the moments neither overflow nor underflow.
// The samples are K8's (generated form: mag_sample, regenerated in each pass) or read from memory (fed form).
// Reductions are a fixed butterfly within each warp and the warps in order: a run's result depends only on
// its samples, whatever the batch, run_offset or sharding.  A singular 3x3 or 4x4 system (a pivot at or below
// kMagCalSingTol * max|A|, or a NaN), or any non-finite output (a non-finite sample, overflowing moments), gives
// NaN in all 13 outputs of the run and in its mag_cal rows.  Spec: oracle/magcal_np.py (calibrate_moments);
// exact reference and rounding bound: oracle/magcal_exact.py; DESIGN.md section 3.11.
#pragma once
#include "common.cuh"
#include "mag_kernel.cuh"

namespace b2ins {

constexpr int kMagCalThreads = 256;
constexpr int kMagCalMoments = 19;       // sum d [3], sum d d^T [6] (xx xy xz yy yz zz), cubic [10]
constexpr double kMagCalSingTol = 1e-12;

struct MagCalParams {
  int64_t runs, n;
  int64_t seg[6];            // (x0, xf, y0, yf, z0, zf), half-open, each >= 3 rows inside [0, n)
  // generated form (K8's model and draws)
  int64_t run_offset;
  const double* ref;         // [n][3]
  double si[9], hi[3], std[3];
  uint32_t k0, k1;
  // fed form: sample k of run r at x[r * run_stride + k * sample_stride + c]
  const double* x;
  int64_t run_stride, sample_stride;
  double* soft_iron;         // [runs][9] row-major
  double* hard_iron;         // [runs][4]
  double* err;               // [runs][13] or null (generated form): E (9), e_hi (3), e_r
  double* mag_cal;           // [runs][sum of lengths][3] or null (fed form): S m - hard_iron[0:3]
};

template <bool kFed>
__device__ __forceinline__ void magcal_sample(const MagCalParams& p, int64_t r, int64_t k, double m[3]) {
  if constexpr (kFed) {
    const double* s = p.x + r * p.run_stride + k * p.sample_stride;
    m[0] = s[0];
    m[1] = s[1];
    m[2] = s[2];
  } else {
    const uint64_t run = static_cast<uint64_t>(p.run_offset + r);
    mag_sample(p.ref, p.si, p.hi, p.std, k, static_cast<uint32_t>(run), static_cast<uint32_t>(run >> 32), p.k0,
               p.k1, m);
  }
}

__device__ __forceinline__ double min_nan(double a, double b) { return (a < b || a != a) ? a : b; }

// x <- A^-1 x by Gaussian elimination with partial pivoting (oracle magcal_np.solve); false when singular
template <int N>
__device__ bool magcal_solve(double (&A)[N][N], double (&x)[N]) {
  double amax = 0.0;
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = 0; j < N; ++j) amax = max_nan(amax, fabs(A[i][j]));
#pragma unroll
  for (int c = 0; c < N; ++c) {
    int p = c;
#pragma unroll
    for (int r = c + 1; r < N; ++r)
      if (fabs(A[r][c]) > fabs(A[p][c])) p = r;
    if (!(fabs(A[p][c]) > kMagCalSingTol * amax)) return false;
    if (p != c) {
#pragma unroll
      for (int j = 0; j < N; ++j) {
        const double t = A[c][j];
        A[c][j] = A[p][j];
        A[p][j] = t;
      }
      const double t = x[c];
      x[c] = x[p];
      x[p] = t;
    }
#pragma unroll
    for (int r = c + 1; r < N; ++r) {
      const double f = A[r][c] / A[c][c];
#pragma unroll
      for (int j = c; j < N; ++j) A[r][j] -= f * A[c][j];
      x[r] -= f * x[c];
    }
  }
#pragma unroll
  for (int c = N - 1; c >= 0; --c) {
    double s = 0.0;
#pragma unroll
    for (int j = c + 1; j < N; ++j) s += A[c][j] * x[j];
    x[c] = (x[c] - s) / A[c][c];
  }
  return true;
}

// The CTA's sum of v[0..K) (warp butterfly, then the warps in order) into out[0..K) (shared); red: [8][K] shared
template <int K>
__device__ __forceinline__ void magcal_block_sum(double (&v)[K], double* red, double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < K; ++i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < K; ++i) red[warp * K + i] = v[i];
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double s = red[threadIdx.x];
    for (int w = 1; w < kMagCalThreads / 32; ++w) s += red[w * K + threadIdx.x];
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

// The plane-fit normal of one segment from its moments (N rows, shift t): the reference's sign rule (largest
// magnitude component positive) and normalisation; false when the 3x3 system is singular
__device__ bool magcal_normal(const double* mom, double N, const double t[3], double v[3]) {
  const double* s1 = mom;
  const double* q = mom + 3;
  const int qi[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
  double A[3][3], x[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) A[i][j] = ((q[qi[i][j]] + t[i] * s1[j]) + s1[i] * t[j]) + N * (t[i] * t[j]);
    x[i] = s1[i] + N * t[i];
  }
  if (!magcal_solve<3>(A, x)) return false;
  int im = 0;
  if (fabs(x[1]) > fabs(x[im])) im = 1;
  if (fabs(x[2]) > fabs(x[im])) im = 2;
  const double sg = x[im] < 0.0 ? -1.0 : 1.0;
  const double nrm = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
#pragma unroll
  for (int i = 0; i < 3; ++i) v[i] = (sg * x[i]) / nrm;
  return true;
}

template <bool kFed>
__global__ void __launch_bounds__(kMagCalThreads) magcal_kernel(const __grid_constant__ MagCalParams p) {
  __shared__ double red[(kMagCalThreads / 32) * kMagCalMoments];
  __shared__ double mom[3][kMagCalMoments];
  __shared__ double ext[3][4];             // per segment: max a, min a, max b, min b
  __shared__ double O[9], sens[3], hard[4];
  const int64_t r = blockIdx.x;
  double t[3];
  magcal_sample<kFed>(p, r, p.seg[0], t);

  // pass 1: moments of d = m - t
  for (int sgi = 0; sgi < 3; ++sgi) {
    double acc[kMagCalMoments];
#pragma unroll
    for (int i = 0; i < kMagCalMoments; ++i) acc[i] = 0.0;
    for (int64_t k = p.seg[2 * sgi] + threadIdx.x; k < p.seg[2 * sgi + 1]; k += kMagCalThreads) {
      double m[3];
      magcal_sample<kFed>(p, r, k, m);
      const double d0 = m[0] - t[0], d1 = m[1] - t[1], d2 = m[2] - t[2];
      const double xx = d0 * d0, xy = d0 * d1, xz = d0 * d2, yy = d1 * d1, yz = d1 * d2, zz = d2 * d2;
      acc[0] += d0;
      acc[1] += d1;
      acc[2] += d2;
      acc[3] += xx;
      acc[4] += xy;
      acc[5] += xz;
      acc[6] += yy;
      acc[7] += yz;
      acc[8] += zz;
      acc[9] += xx * d0;
      acc[10] += xx * d1;
      acc[11] += xx * d2;
      acc[12] += xy * d1;
      acc[13] += xy * d2;
      acc[14] += xz * d2;
      acc[15] += yy * d1;
      acc[16] += yy * d2;
      acc[17] += yz * d2;
      acc[18] += zz * d2;
    }
    magcal_block_sum<kMagCalMoments>(acc, red, mom[sgi]);
  }

  // the normals: the rows of O (NaN when a system is singular)
  if (threadIdx.x == 0) {
    bool ok = true;
    for (int sgi = 0; sgi < 3; ++sgi)
      ok = magcal_normal(mom[sgi], static_cast<double>(p.seg[2 * sgi + 1] - p.seg[2 * sgi]), t, O + 3 * sgi) && ok;
    if (!ok)
      for (int i = 0; i < 9; ++i) O[i] = __longlong_as_double(0x7ff8000000000000ll);
  }
  __syncthreads();

  // pass 2: extremes of the two columns of c = O m each segment's sensitivity needs
  const int cols[3][2] = {{2, 1}, {2, 0}, {1, 0}};
  for (int sgi = 0; sgi < 3; ++sgi) {
    const double* oa = O + 3 * cols[sgi][0];
    const double* ob = O + 3 * cols[sgi][1];
    const double a0 = oa[0], a1 = oa[1], a2 = oa[2], b0 = ob[0], b1 = ob[1], b2 = ob[2];
    double ex[4] = {-INFINITY, INFINITY, -INFINITY, INFINITY};
    for (int64_t k = p.seg[2 * sgi] + threadIdx.x; k < p.seg[2 * sgi + 1]; k += kMagCalThreads) {
      double m[3];
      magcal_sample<kFed>(p, r, k, m);
      const double ca = a0 * m[0] + a1 * m[1] + a2 * m[2];
      const double cb = b0 * m[0] + b1 * m[1] + b2 * m[2];
      ex[0] = max_nan(ex[0], ca);
      ex[1] = min_nan(ex[1], ca);
      ex[2] = max_nan(ex[2], cb);
      ex[3] = min_nan(ex[3], cb);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ex[0] = max_nan(ex[0], __shfl_xor_sync(0xffffffffu, ex[0], o));
      ex[1] = min_nan(ex[1], __shfl_xor_sync(0xffffffffu, ex[1], o));
      ex[2] = max_nan(ex[2], __shfl_xor_sync(0xffffffffu, ex[2], o));
      ex[3] = min_nan(ex[3], __shfl_xor_sync(0xffffffffu, ex[3], o));
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i) red[(threadIdx.x >> 5) * 4 + i] = ex[i];
    }
    __syncthreads();
    if (threadIdx.x < 4) {
      double e = red[threadIdx.x];
      for (int w = 1; w < kMagCalThreads / 32; ++w)
        e = (threadIdx.x & 1) ? min_nan(e, red[w * 4 + threadIdx.x]) : max_nan(e, red[w * 4 + threadIdx.x]);
      ext[sgi][threadIdx.x] = e;
    }
    __syncthreads();
  }

  // the sensitivities, S and the sphere fit in the shifted calibrated frame u = S d
  if (threadIdx.x == 0) {
    const double sZ2Y = (ext[0][0] - ext[0][1]) / (ext[0][2] - ext[0][3]);
    const double sZ2X = (ext[1][0] - ext[1][1]) / (ext[1][2] - ext[1][3]);
    const double sY2X = (ext[2][0] - ext[2][1]) / (ext[2][2] - ext[2][3]);
    const double s[3] = {1.0, 1.0 / sY2X, (1.0 + sY2X * sY2X) / (sY2X * sY2X * sZ2X + sY2X * sZ2Y)};
    double Sm[3][3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Sm[i][j] = s[i] * O[3 * i + j];
    // the moments of all three segments
    double D[kMagCalMoments];
    for (int i = 0; i < kMagCalMoments; ++i) D[i] = (mom[0][i] + mom[1][i]) + mom[2][i];
    const double N = static_cast<double>((p.seg[1] - p.seg[0]) + (p.seg[3] - p.seg[2]) + (p.seg[5] - p.seg[4]));
    const int qi[3][3] = {{3, 4, 5}, {4, 6, 7}, {5, 7, 8}};
    // cubic index of (a, b, c), a <= b <= c: xxx xxy xxz xyy xyz xzz yyy yyz yzz zzz
    const int ci[3][3][3] = {{{9, 10, 11}, {10, 12, 13}, {11, 13, 14}},
                             {{10, 12, 13}, {12, 15, 16}, {13, 16, 17}},
                             {{11, 13, 14}, {13, 16, 17}, {14, 17, 18}}};
    double U1[3], SD[3][3], U2[3][3], G[3][3], w[3], v[3];
    for (int i = 0; i < 3; ++i) {
      U1[i] = (Sm[i][0] * D[0] + Sm[i][1] * D[1]) + Sm[i][2] * D[2];
      for (int j = 0; j < 3; ++j) {
        SD[i][j] = (Sm[i][0] * D[qi[0][j]] + Sm[i][1] * D[qi[1][j]]) + Sm[i][2] * D[qi[2][j]];
        G[i][j] = (Sm[0][i] * Sm[0][j] + Sm[1][i] * Sm[1][j]) + Sm[2][i] * Sm[2][j];   // S^T S
      }
    }
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) U2[i][j] = (SD[i][0] * Sm[j][0] + SD[i][1] * Sm[j][1]) + SD[i][2] * Sm[j][2];
    // sum u_i |u|^2 = (S w)_i, w_a = sum_bc (S^T S)_bc D3_abc
    for (int a = 0; a < 3; ++a) {
      double acc = 0.0;
      for (int b = 0; b < 3; ++b)
        for (int c = 0; c < 3; ++c) acc += G[b][c] * D[ci[a][b][c]];
      w[a] = acc;
    }
    for (int i = 0; i < 3; ++i) v[i] = (Sm[i][0] * w[0] + Sm[i][1] * w[1]) + Sm[i][2] * w[2];
    // the fit on f u, f = 2^-e, e = floor((e_tr - e_N) / 2) from the binary exponents of trace(sum u u^T) and N,
    // so f is within a factor 2 of 1 / rms |u|: every entry of HH is then on the scale of N, the pivot rule does
    // not depend on the units of the samples, and every scaling is exact (no division or root on the way)
    const double tr = (U2[0][0] + U2[1][1]) + U2[2][2];
    int e = 0;
    if (isfinite(tr) && tr > 0.0) {
      int etr, en;
      frexp(tr, &etr);
      frexp(N, &en);
      e = (etr - en) >> 1;
    }
    const double f = ldexp(1.0, -e), f2 = f * f, g = ldexp(1.0, e), g2 = g * g;   // g = 1 / f
    double HH[4][4], q[4];
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) HH[i][j] = (4.0 * U2[i][j]) * f2;
      HH[i][3] = HH[3][i] = (2.0 * U1[i]) * f;
      q[i] = (2.0 * v[i]) * (f2 * f);
    }
    HH[3][3] = N;
    q[3] = tr * f2;
    bool ok = magcal_solve<4>(HH, q) && !isnan(O[0]);
    double out[13];
    for (int i = 0; i < 3; ++i) {
      const double T = (Sm[i][0] * t[0] + Sm[i][1] * t[1]) + Sm[i][2] * t[2];
      q[i] *= g;
      out[9 + i] = q[i] + T;
      for (int j = 0; j < 3; ++j) out[3 * i + j] = Sm[i][j];
    }
    q[3] *= g2;
    out[12] = sqrt(q[3] + ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]));
    for (int i = 0; i < 13; ++i) ok = ok && isfinite(out[i]);
    if (!ok)
      for (int i = 0; i < 13; ++i) out[i] = __longlong_as_double(0x7ff8000000000000ll);
    for (int i = 0; i < 9; ++i) p.soft_iron[r * 9 + i] = out[i];
    for (int i = 0; i < 3; ++i) sens[i] = s[i];
    for (int i = 0; i < 4; ++i) {
      p.hard_iron[r * 4 + i] = out[9 + i];
      hard[i] = out[9 + i];
    }
    if (!kFed && p.err) {   // against the truth: k = trace(S si) / 3, E = S si / k - I, hard_iron / k - (hi, |b|)
      double P[3][3];
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) P[i][j] = (out[3 * i] * p.si[j] + out[3 * i + 1] * p.si[3 + j]) + out[3 * i + 2] * p.si[6 + j];
      const double k = ((P[0][0] + P[1][1]) + P[2][2]) / 3.0;
      double* e = p.err + r * 13;
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) e[3 * i + j] = P[i][j] / k - (i == j ? 1.0 : 0.0);
      for (int i = 0; i < 3; ++i) e[9 + i] = out[9 + i] / k - p.hi[i];
      const double bn = sqrt((p.ref[0] * p.ref[0] + p.ref[1] * p.ref[1]) + p.ref[2] * p.ref[2]);
      e[12] = out[12] / k - bn;
    }
  }
  if (!kFed || p.mag_cal == nullptr) return;
  __syncthreads();

  // pass 3 (fed form, on request): mag_cal, the reference's staged corrections O m, diag(s) ., - hard_iron
  int64_t row = 0;
  double* outc = p.mag_cal + r * 3 * ((p.seg[1] - p.seg[0]) + (p.seg[3] - p.seg[2]) + (p.seg[5] - p.seg[4]));
  for (int sgi = 0; sgi < 3; ++sgi) {
    const int64_t a = p.seg[2 * sgi], b = p.seg[2 * sgi + 1];
    for (int64_t k = a + threadIdx.x; k < b; k += kMagCalThreads) {
      double m[3];
      magcal_sample<kFed>(p, r, k, m);
      double* o = outc + (row + k - a) * 3;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const double c = O[3 * i] * m[0] + O[3 * i + 1] * m[1] + O[3 * i + 2] * m[2];
        o[i] = sens[i] * c - hard[i];
      }
    }
    row += b - a;
  }
}

}  // namespace b2ins
