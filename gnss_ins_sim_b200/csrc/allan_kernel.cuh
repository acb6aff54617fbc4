// K4: non-overlapped Allan variance on cluster sizes m = j*10^k (j = 1..9) --
// allan.allan_var, allan/allan.py:18-59.
//
// All clusters start at sample 0, so a cluster of 10m samples is the union of 10 clusters
// of m samples.  Level k works on the decade sums S_k (S_0 = x, S_{k+1}[i] = sum of
// S_k[10i..10i+9]) and yields the nine cluster sizes j*10^k plus S_{k+1}; the series is
// read from HBM once (level 0) instead of once per tau as the reference does.
//
// A tile is one (series, chunk) pair; a chunk is kAllanChunk = 2*2520 level-k elements
// (2520 = lcm(1..10): every cluster size starts a cluster at each chunk start) plus a
// 9-element halo for the cluster that ends where the chunk starts.  Every successive-difference
// term is the difference of two cluster sums formed directly from the samples of its two bins, so
// a non-finite sample reaches only the terms whose bins hold it, as in the reference.  Where a
// tile subtracts an offset (its first element, which cancels in every difference), it uses it
// only when it is finite: an infinite offset would turn every term of the tile into inf - inf.
#pragma once
#include <cstring>

#include "common.cuh"
#include "mc_kernel.cuh"   // TriadNoise: the pre-digested error model of the generating front end

namespace b2ins {

constexpr int kAllanChunk = 5040;
constexpr int kAllanHalo = 9;
constexpr int kAllanMaxLevels = 10;

struct AllanLevelParams {
  int64_t len;           // N_k: elements of this level per series
  int64_t next_len;      // N_{k+1} = N_k / 10 (0: do not produce)
  int64_t nseries;
  const double* src;     // level 0: x ; else S_k [nseries][len]
  int64_t inner, outer_stride, sample_stride;  // level 0 addressing
  int level0;
  double* next;          // S_{k+1} [nseries][next_len]
  double* partial;       // [nseries][chunks][9]
  int64_t chunks;        // chunks per series at this level
  int jmax;              // cluster multipliers 1..jmax are wanted at this level
  int64_t chunk_first;   // this launch covers chunks [chunk_first, chunk_first + chunk_count)
  int64_t chunk_count;
  int64_t src_pitch;     // row pitch of S_k (levels >= 1) and of S_{k+1}: even, so that rows are
  int64_t next_pitch;    // 16-byte aligned for the bulk copies
};

// ---- fast path: FULL chunks ---------------------------------------------------------------
// A full chunk holds an integer number of clusters of every size (5040 = 2 lcm(1..10)), so the
// cluster sums are built hierarchically IN REGISTERS, without bound checks, by three kinds of work
// items (16 warps; every sample is read from shared memory once per kind):
//   X (105 items of 48 samples, 4 warps): j = 2, 4, 8      (pairs, pairs of pairs, ...)
//   Y (280 items of 18 samples, 9 warps): j = 1, 3, 6, 9   (triples, pairs / triples of triples)
//   C ( 72 items of 70 samples, 3 warps): j = 5, 7 and the decade sums that feed the next level
// (~10 FP64 instructions per sample in all).  An item is read with 128-bit shared-memory loads;
// they are conflict-free when the item pitch is an odd number of 16-byte units: 9 and 35 for Y and
// C, which read the raw tile where the copy engine put it and subtract the tile offset in
// registers, while X (24 units) reads a copy padded 48 -> 50 doubles, offset-subtracted when it is
// made.  The difference that straddles the left edge of an item is formed from the (at most 9)
// samples to the left of the item, which are in shared memory too (the halo for item 0): no
// exchange between threads, no barrier.  Two front ends:
//   allan_stream_kernel  contiguous, 16-byte aligned series: persistent CTA per SM; the raw tile
//                        arrives by one TMA bulk copy into a three-slot ring (two tiles in
//                        flight behind the one being computed), the padded copy and the block
//                        reduction are double-buffered: ONE __syncthreads per tile;
//   allan_full_kernel    any stride / alignment: per-thread loads, one tile per CTA.
// Both take the ragged last chunk of a series with the masked form of the same work items.
constexpr int kAllanItemsX = kAllanChunk / 48;    // 105
constexpr int kAllanItemsY = kAllanChunk / 18;    // 280
constexpr int kAllanItemsC = kAllanChunk / 70;    // 72
constexpr int kAllanWarpsX = 4, kAllanWarpsY = 9, kAllanWarpsC = 3;
constexpr int kAllanFastWarps = kAllanWarpsX + kAllanWarpsY + kAllanWarpsC;   // 16
constexpr int kAllanFastThreads = 32 * kAllanFastWarps;   // 512
constexpr int kAllanLead = kAllanHalo + 1;        // 10: chunk element e lives at raw[10 + e]
constexpr int kAllanRawLen = 5056;                // >= 10 + 5040, a multiple of 2
constexpr int kAllanPadLead = 12;                 // halo element -k lives at pad[-2 - k]
constexpr int kAllanPadLen = kAllanPadLead + kAllanItemsX * 50 + 2;   // 5264

__device__ __forceinline__ double sq_acc(double a, double b, double acc) {
  const double d = a - b;
  return fma(d, d, acc);
}

// sum over i = 1..N-1 of (c[i] - c[i-1])^2 in interleaved accumulators (the serial FMA chain of a
// single accumulator would cost 8 cycles per link)
template <int N>
__device__ __forceinline__ double sum_sq_diff(const double (&c)[N]) {
  double a[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for (int i = 1; i < N; ++i) a[i & 3] = sq_acc(c[i], c[i - 1], a[i & 3]);
  return (a[0] + a[1]) + (a[2] + a[3]);
}

// The same with a validity mask for the ragged last chunk of a series: cluster i ends (exclusive)
// at local element end0 + i * step and counts only if that is within lim (the elements of the
// chunk covered by COMPLETE clusters of this size).  Selects, not multiplications: what lies
// beyond the end of the series in shared memory is stale data.
template <int N, bool RAGGED>
__device__ __forceinline__ double sum_sq_diff_m(const double (&c)[N], int end0, int step, int lim) {
  if (!RAGGED) return sum_sq_diff(c);
  double a[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for (int i = 1; i < N; ++i) {
    const double t = sq_acc(c[i], c[i - 1], a[i & 3]);
    a[i & 3] = (end0 + i * step <= lim) ? t : a[i & 3];
  }
  return (a[0] + a[1]) + (a[2] + a[3]);
}
template <bool RAGGED>
__device__ __forceinline__ double sq_acc_m(double a, double b, double acc, int end, int lim) {
  const double t = sq_acc(a, b, acc);
  return (!RAGGED || end <= lim) ? t : acc;
}

// Warp totals of four values per lane in 5 packed butterfly steps; lane L returns the total of
// value number L >> 3.  Fixed pairing: deterministic.
__device__ __forceinline__ double warp_sum4(double v0, double v1, double v2, double v3, int lane) {
  const bool up16 = lane & 16;
  const double w0 = (up16 ? v2 : v0) + __shfl_xor_sync(0xffffffffu, up16 ? v0 : v2, 16);
  const double w1 = (up16 ? v3 : v1) + __shfl_xor_sync(0xffffffffu, up16 ? v1 : v3, 16);
  const bool up8 = lane & 8;
  double t = (up8 ? w1 : w0) + __shfl_xor_sync(0xffffffffu, up8 ? w0 : w1, 8);
  t += __shfl_xor_sync(0xffffffffu, t, 4);
  t += __shfl_xor_sync(0xffffffffu, t, 2);
  t += __shfl_xor_sync(0xffffffffu, t, 1);
  return t;
}

// One tile.  in: the raw tile as loaded (NOT offset-subtracted), chunk element e at in[10 + e],
// halo at in[1..9]; pad: X's copy (subtracted), element e at pad[e + 2 (e / 48)], halo element -k
// at pad[-2 - k].  Returns the thread's sums of squared differences in v[0..3]; no barrier inside.
// SUB: subtract the tile offset (the first element of the tile) from every sample before it is
// used.  It cancels in every difference; removing it keeps the rounding of the cluster sums at
// the level of the signal's VARIATION instead of its magnitude, which matters for the decade sums
// of the upper levels (magnitude ~ 10^k, variation ~ 10^(k/2)).  Level 0 adds at most 10 raw
// samples per cluster and skips it (off = 0 there, and X's copy is made unsubtracted).
// RAGGED: the last chunk of a series (fewer than 5040 elements): every term is masked by the
// number of elements its cluster size covers with complete clusters.
template <bool SUB, bool RAGGED>
__device__ __forceinline__ void allan_tile_compute(const AllanLevelParams& p, int64_t series, int64_t chunk,
                                                   const double* in, const double* pad, double off,
                                                   double (&v)[4]) {
  const int tid = threadIdx.x, warp = tid >> 5;
  constexpr int kW1 = kAllanWarpsX, kW2 = kW1 + kAllanWarpsY;
  const int role = (warp >= kW1) + (warp >= kW2);
  const int item = tid - 32 * (role == 0 ? 0 : role == 1 ? kW1 : kW2);
  const bool left = item > 0 || chunk != 0;   // the item has a left neighbour in this series
  const double* x = in + kAllanLead;
  // elements of this chunk covered by complete clusters of size j (only used when RAGGED)
  const int64_t c0 = chunk * kAllanChunk;
  auto lim = [&](int j) { return RAGGED ? static_cast<int>((p.len / j) * j - c0) : kAllanChunk; };
  double v0 = 0.0, v1 = 0.0, v2 = 0.0, v3 = 0.0;   // the role's sums of squared differences
  if (role == 0) {
    if (item < kAllanItemsX) {   // j = 2, 4, 8: the 8 samples to the left, then two blocks of 24
      const double2* src = reinterpret_cast<const double2*>(pad + 50 * item);
      const int l2 = lim(2), l4 = lim(4), l8 = lim(8);
      double pP, pQ, pO;
      {
        const double2 t0 = src[-5], t1 = src[-4], t2 = src[-3], t3 = src[-2];
        pP = t3.x + t3.y;
        pQ = (t2.x + t2.y) + pP;
        pO = ((t0.x + t0.y) + (t1.x + t1.y)) + pQ;
      }
#pragma unroll
      for (int sb = 0; sb < 2; ++sb) {
        double P[12], Q[6], O[3];
#pragma unroll
        for (int i = 0; i < 12; ++i) {
          const double2 t = src[12 * sb + i];
          P[i] = t.x + t.y;
        }
#pragma unroll
        for (int i = 0; i < 6; ++i) Q[i] = P[2 * i] + P[2 * i + 1];
#pragma unroll
        for (int i = 0; i < 3; ++i) O[i] = Q[2 * i] + Q[2 * i + 1];
        const int eb = 48 * item + 24 * sb;
        if (sb > 0 || left) {
          v0 = sq_acc_m<RAGGED>(P[0], pP, v0, eb + 2, l2);
          v1 = sq_acc_m<RAGGED>(Q[0], pQ, v1, eb + 4, l4);
          v2 = sq_acc_m<RAGGED>(O[0], pO, v2, eb + 8, l8);
        }
        v0 += sum_sq_diff_m<12, RAGGED>(P, eb + 2, 2, l2);
        v1 += sum_sq_diff_m<6, RAGGED>(Q, eb + 4, 4, l4);
        v2 += sum_sq_diff_m<3, RAGGED>(O, eb + 8, 8, l8);
        pP = P[11]; pQ = Q[5]; pO = O[2];
      }
    }
  } else if (role == 1) {
    if (item < kAllanItemsY) {   // j = 1, 3, 6, 9: the 9 samples to the left, then 18 samples
      const double* xs = x + 18 * item;
      const double2* src = reinterpret_cast<const double2*>(xs);
      double y[18], T[6], S[3], N[2];
#pragma unroll
      for (int i = 0; i < 9; ++i) {
        const double2 t = src[i];
        y[2 * i] = SUB ? t.x - off : t.x;
        y[2 * i + 1] = SUB ? t.y - off : t.y;
      }
      double py, pT, pS, pN;
      {
        double l[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) l[k] = SUB ? xs[k - 9] - off : xs[k - 9];
        py = l[8];
        pT = (l[6] + l[7]) + l[8];
        const double t1 = (l[3] + l[4]) + l[5], t0 = (l[0] + l[1]) + l[2];
        pS = t1 + pT;
        pN = (t0 + t1) + pT;
      }
#pragma unroll
      for (int i = 0; i < 6; ++i) T[i] = (y[3 * i] + y[3 * i + 1]) + y[3 * i + 2];
#pragma unroll
      for (int i = 0; i < 3; ++i) S[i] = T[2 * i] + T[2 * i + 1];
#pragma unroll
      for (int i = 0; i < 2; ++i) N[i] = (T[3 * i] + T[3 * i + 1]) + T[3 * i + 2];
      const int e0 = 18 * item;
      const int l1 = lim(1), l3 = lim(3), l6 = lim(6), l9 = lim(9);
      v0 = sum_sq_diff_m<6, RAGGED>(T, e0 + 3, 3, l3);
      v1 = sum_sq_diff_m<3, RAGGED>(S, e0 + 6, 6, l6);
      v2 = sum_sq_diff_m<2, RAGGED>(N, e0 + 9, 9, l9);
      v3 = sum_sq_diff_m<18, RAGGED>(y, e0 + 1, 1, l1);
      if (left) {
        v0 = sq_acc_m<RAGGED>(T[0], pT, v0, e0 + 3, l3);
        v1 = sq_acc_m<RAGGED>(S[0], pS, v1, e0 + 6, l6);
        v2 = sq_acc_m<RAGGED>(N[0], pN, v2, e0 + 9, l9);
        v3 = sq_acc_m<RAGGED>(y[0], py, v3, e0 + 1, l1);
      }
    }
  } else {
    if (item < kAllanItemsC) {   // j = 5, 7 and the decade sums: the 7 samples to the left, then 70
      const double* xs = x + 70 * item;
      const double2* src = reinterpret_cast<const double2*>(xs);
      double* nx = p.next + series * p.next_pitch + (chunk * kAllanChunk) / 10 + 7 * item;
      const double off10 = SUB ? 10.0 * off : 0.0;
      const int l5 = lim(5), l7 = lim(7), l10 = lim(10);
      double pF, pG;
      {
        double l[7];
#pragma unroll
        for (int k = 0; k < 7; ++k) l[k] = SUB ? xs[k - 7] - off : xs[k - 7];
        pF = ((l[2] + l[3]) + (l[4] + l[5])) + l[6];
        pG = ((l[0] + l[1]) + (l[2] + l[3])) + ((l[4] + l[5]) + l[6]);
      }
      // the 70 samples stream through in blocks of 10 (fives, decades); the sevens are gathered
      // from a 14-sample window that slides over the blocks (all indices are compile-time)
      double w[14];   // samples 14 g .. 14 g + 13 of the current seven-pair g
#pragma unroll
      for (int sb = 0; sb < 7; ++sb) {
        double y[10];
#pragma unroll
        for (int i = 0; i < 5; ++i) {
          const double2 t = src[5 * sb + i];
          y[2 * i] = SUB ? t.x - off : t.x;
          y[2 * i + 1] = SUB ? t.y - off : t.y;
        }
        const double F0 = ((y[0] + y[1]) + (y[2] + y[3])) + y[4];
        const double F1 = ((y[5] + y[6]) + (y[7] + y[8])) + y[9];
        const int eb = 70 * item + 10 * sb;
        if (sb > 0 || left) v0 = sq_acc_m<RAGGED>(F0, pF, v0, eb + 5, l5);
        v0 = sq_acc_m<RAGGED>(F1, F0, v0, eb + 10, l5);
        pF = F1;
        if (p.next_len > 0 && (!RAGGED || eb + 10 <= l10)) nx[sb] = (F0 + F1) + off10;
#pragma unroll
        for (int i = 0; i < 10; ++i) {
          const int e = 10 * sb + i;      // sample index in the item
          w[e % 14] = y[i];
          if (e % 14 == 13) {             // a pair of sevens is complete
            const double G0 = ((w[0] + w[1]) + (w[2] + w[3])) + ((w[4] + w[5]) + w[6]);
            const double G1 = ((w[7] + w[8]) + (w[9] + w[10])) + ((w[11] + w[12]) + w[13]);
            if (e > 13 || left) v1 = sq_acc_m<RAGGED>(G0, pG, v1, 70 * item + e - 6, l7);
            v1 = sq_acc_m<RAGGED>(G1, G0, v1, 70 * item + e + 1, l7);
            pG = G1;
          }
        }
      }
    }
  }
  v[0] = v0; v[1] = v1; v[2] = v2; v[3] = v3;
}

// one packed butterfly per warp; allan_tile_fold adds the role's warps in order after a barrier
__device__ __forceinline__ void allan_tile_reduce(const double (&v)[4], double (*red)[4]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double t = warp_sum4(v[0], v[1], v[2], v[3], lane);
  if ((lane & 7) == 0) red[warp][lane >> 3] = t;
}

// threads 0..8, after a barrier behind allan_tile_compute: partial sums of the chunk for j = tid+1
__device__ __forceinline__ void allan_tile_fold(const AllanLevelParams& p, int64_t series, int64_t chunk,
                                                const double (*red)[4]) {
  const int tid = threadIdx.x;
  constexpr int kW1 = kAllanWarpsX, kW2 = kW1 + kAllanWarpsY;
  // j = tid + 1 is held by role {1,0,1,0,2,1,2,0,1}[tid] in column {3,0,0,1,0,1,1,2,2}[tid]
  const int r = static_cast<int>((0x102120101ull >> (4 * tid)) & 15);
  const int c = static_cast<int>((0x221101003ull >> (4 * tid)) & 15);
  const int w0 = r == 0 ? 0 : r == 1 ? kW1 : kW2;
  const int w1 = r == 0 ? kW1 : r == 1 ? kW2 : kAllanFastWarps;
  double v = 0.0;
#pragma unroll
  for (int w = 0; w < kAllanWarpsY; ++w)
    if (w0 + w < w1) v += red[w0 + w][c];
  p.partial[(series * p.chunks + chunk) * 9 + tid] = (tid < p.jmax) ? v : 0.0;
}

template <bool UNIT>   // UNIT: consecutive samples are adjacent in memory
__global__ void __launch_bounds__(kAllanFastThreads, 2) allan_full_kernel(const __grid_constant__ AllanLevelParams p) {
  extern __shared__ __align__(128) double smem[];
  double* in = smem;                                   // [kAllanRawLen] raw tile, as loaded
  double* pad = smem + kAllanRawLen + kAllanPadLead;   // X's padded, offset-subtracted copy
  __shared__ double red[kAllanFastWarps][4];
  const int64_t series = blockIdx.x / p.chunk_count;
  const int64_t chunk = p.chunk_first + blockIdx.x % p.chunk_count;
  const int64_t c0 = chunk * kAllanChunk;
  const bool has_prev = chunk != 0;
  const int tid = threadIdx.x;
  const double* base;
  int64_t stride;
  if (p.level0) {
    base = p.src + (series / p.inner) * p.outer_stride + (series % p.inner);
    stride = UNIT ? 1 : p.sample_stride;
  } else {
    base = p.src + series * p.src_pitch;
    stride = 1;
  }
  const double off0 = p.level0 ? 0.0 : base[(c0 - (has_prev ? kAllanHalo : 0)) * stride];
  const double off = isfinite(off0) ? off0 : 0.0;
  const bool ragged = c0 + kAllanChunk > p.len;
  const int cnt = ragged ? static_cast<int>(p.len - c0) : kAllanChunk;   // elements of the chunk
  {
    // loaders: thread (g, pos) loads element 48 (7 q + g) + pos in pass q; every load is issued
    // before the first use (15 independent requests in flight per thread)
    constexpr int kLoaders = 336;   // 7 blocks of 48 per pass, 15 passes
    constexpr int kPasses = 15;
    const int g = tid / 48, pos = tid - 48 * g;
    const double* src = base + (c0 + 48 * g + pos) * stride;
    double v[kPasses];
    double hv = 0.0;
    if (tid < kLoaders) {
#pragma unroll
      for (int q = 0; q < kPasses; ++q)
        v[q] = (48 * (7 * q + g) + pos < cnt) ? src[static_cast<int64_t>(q) * kLoaders * stride] : 0.0;
    } else if (has_prev && tid < kLoaders + kAllanHalo) {
      hv = base[(c0 - kAllanHalo + (tid - kLoaders)) * stride];
    }
    if (tid < kLoaders) {
      double* xr = in + kAllanLead + 48 * g + pos;
      double* xp = pad + 50 * g + pos;
#pragma unroll
      for (int q = 0; q < kPasses; ++q) {
        xr[q * kLoaders] = v[q];
        xp[q * 7 * 50] = v[q] - off;   // off = 0 at level 0
      }
    } else if (tid < kLoaders + kAllanHalo) {
      const int k = kAllanHalo - (tid - kLoaders);   // halo element -k, k = 9..1
      in[kAllanLead - k] = hv;                       // zeros without a left neighbour (unused)
      pad[-2 - k] = hv - off;
    }
  }
  __syncthreads();
  double acc[4];
  if (p.level0) {
    if (ragged)
      allan_tile_compute<false, true>(p, series, chunk, in, pad, 0.0, acc);
    else
      allan_tile_compute<false, false>(p, series, chunk, in, pad, 0.0, acc);
  } else {
    if (ragged)
      allan_tile_compute<true, true>(p, series, chunk, in, pad, off, acc);
    else
      allan_tile_compute<true, false>(p, series, chunk, in, pad, off, acc);
  }
  allan_tile_reduce(acc, red);
  __syncthreads();
  if (tid < 9) allan_tile_fold(p, series, chunk, red);
}

// Persistent front end: CTA b takes tiles b, b + grid, ...
constexpr int kAllanStages = 3;
template <bool SUB>
__global__ void __launch_bounds__(kAllanFastThreads, 1) allan_stream_kernel(const __grid_constant__ AllanLevelParams p) {
  extern __shared__ __align__(128) double smem[];
  double* in_buf = smem;                                          // [kAllanStages][kAllanRawLen]
  double* pad_buf = smem + kAllanStages * kAllanRawLen;           // [2][kAllanPadLen]
  __shared__ double red[2][kAllanFastWarps][4];
  __shared__ __align__(8) uint64_t full[kAllanStages];
  const int tid = threadIdx.x;
  const int tiles = static_cast<int>(p.nseries * p.chunk_count);   // < 2^31 (checked by the host)
  const int cc = static_cast<int>(p.chunk_count);
  auto issue = [&](int series, int chunk, int slot) {
    const double* base = p.level0 ? p.src + series * p.outer_stride : p.src + series * p.src_pitch;
    const int lead = (chunk != 0) ? kAllanLead : 0;
    const int64_t c0 = static_cast<int64_t>(chunk) * kAllanChunk;
    const int64_t left_in_series = p.len - c0;
    const int cnt = left_in_series < kAllanChunk ? static_cast<int>(left_in_series) : kAllanChunk;
    const int avail = cnt + lead;                      // elements to fetch
    double* dst = in_buf + slot * kAllanRawLen + (kAllanLead - lead);
    const uint32_t bytes = static_cast<uint32_t>((avail & ~1) * sizeof(double));
    if (avail & 1) dst[avail - 1] = base[c0 - lead + avail - 1];   // a bulk copy moves whole 16 B
    mbar_arrive_expect_tx(&full[slot], bytes);
    if (bytes) bulk_g2s(dst, base + c0 - lead, bytes, &full[slot]);
  };
  // (series, chunk) of this CTA's tiles, advanced by gridDim.x tiles at a time without divisions
  const int step_s = static_cast<int>(gridDim.x) / cc, step_c = static_cast<int>(gridDim.x) % cc;
  auto advance = [&](int& series, int& chunk) {
    series += step_s;
    chunk += step_c;
    if (chunk >= cc) {
      chunk -= cc;
      ++series;
    }
  };
  int series = static_cast<int>(blockIdx.x) / cc, chunk = static_cast<int>(blockIdx.x) % cc;
  int fs = series, fc = chunk;   // the tile two ahead (the one to fetch)
  if (tid == 0) {
    for (int s = 0; s < kAllanStages; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
    int tile = blockIdx.x;
    for (int s = 0; s < 2; ++s) {
      if (tile < tiles) issue(fs, fc, s);
      advance(fs, fc);
      tile += gridDim.x;
    }
  }
  __syncthreads();
  int it = 0;
  int prev_series = 0, prev_chunk = 0;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
    const int slot = it % kAllanStages;
    mbar_wait(&full[slot], (it / kAllanStages) & 1);
    const double* in = in_buf + slot * kAllanRawLen;
    double* pad = pad_buf + (it & 1) * kAllanPadLen + kAllanPadLead;
    const double off0 = SUB ? in[chunk != 0 ? 1 : kAllanLead] : 0.0;
    const double off = isfinite(off0) ? off0 : 0.0;
    {
      // X's copy: units of two samples; the five halo units land just below pad[0]
      const double2* in2 = reinterpret_cast<const double2*>(in);
      double2* pad2 = reinterpret_cast<double2*>(pad);
#pragma unroll
      for (int q = 0; q < 5; ++q) {
        const int u = tid + q * kAllanFastThreads;
        if (u < (kAllanLead + kAllanChunk) / 2) {
          double2 w = in2[u];
          if (SUB) {
            w.x -= off;
            w.y -= off;
          }
          const int ue = u - kAllanLead / 2;
          pad2[ue >= 0 ? ue + ue / 24 : ue - 1] = w;
        }
      }
    }
    __syncthreads();   // the only barrier of the tile: pad complete; everybody has finished tile it-1
    if (tid == 0) {    // the slot of tile it-1 is free: fetch tile it+2 into it
      if (tile + 2 * static_cast<int>(gridDim.x) < tiles) {
        fence_async_smem();
        issue(fs, fc, (it + 2) % kAllanStages);
      }
      advance(fs, fc);
    }
    if (it > 0 && tid < 9) allan_tile_fold(p, prev_series, prev_chunk, red[(it - 1) & 1]);
    double acc[4];
    if (static_cast<int64_t>(chunk + 1) * kAllanChunk <= p.len)
      allan_tile_compute<SUB, false>(p, series, chunk, in, pad, off, acc);
    else
      allan_tile_compute<SUB, true>(p, series, chunk, in, pad, off, acc);
    allan_tile_reduce(acc, red[it & 1]);
    prev_series = series;
    prev_chunk = chunk;
    advance(series, chunk);
  }
  __syncthreads();
  if (it > 0 && tid < 9) allan_tile_fold(p, prev_series, prev_chunk, red[(it - 1) & 1]);
}

// ---- K1 fused into level 0: the series is generated in the tile, never written ------------------
// The Allan experiment (Sim + the Allan plugin) used to materialise every run's noisy gyro / accel
// series with K1 (48 B per run-sample) and read them back here: config 4 (256 runs x 14.4 M samples x
// 6 channels) moved 177 GB through HBM twice, in run blocks sized to memory.  This front end replaces
// the bulk copy of the stream kernel by the generator: a persistent CTA owns whole series (series s =
// run s / 6, channel s % 6: accel xyz, gyro xyz -- the Philox draw id of the channel's Box-Muller
// pair), walks its chunks in order and keeps the Gauss-Markov state of the channel in registers, so no
// segment pre-pass is needed.  Thread i of the first 504 makes samples 10 i .. 10 i + 9 of the tile:
// pair (t, channel, run) -> (drift drive, white noise), the zero-state response of its ten drives, and
// an affine scan over the threads (shuffles within a warp, the sixteen warp totals through shared
// memory) gives every thread the drift at the start of its stretch:
//     sample = (ref + b) + w z1 + wd z0 + d[t],   d[t+1] = a d[t] + b_gm z0[t]   (pathgen.py:441-594).
// What leaves the chip at level 0: the decade sums (0.8 B per sample) and nine partials per chunk.
struct AllanGenParams {
  int64_t n, run_offset;
  uint32_t k0, k1;
  TriadNoise gyro, accel;       // pre-digested error models (no vibration in this path)
  const double* ref_gyro;       // [n][3]
  const double* ref_accel;      // [n][3]
};

constexpr int kGenPer = 10;                              // samples per thread and tile
constexpr int kGenThreads = kAllanChunk / kGenPer;       // 504 of the 512 threads generate

__global__ void __launch_bounds__(kAllanFastThreads, 1)
allan_gen_kernel(const __grid_constant__ AllanLevelParams p, const __grid_constant__ AllanGenParams g) {
  extern __shared__ __align__(128) double smem[];
  double* in_buf = smem;                                   // [2][kAllanRawLen]
  double* pad_buf = smem + 2 * kAllanRawLen;               // [2][kAllanPadLen]
  __shared__ double red[2][kAllanFastWarps][4];
  __shared__ double wtot[1][kAllanFastWarps][2];           // (A, E) of every warp's stretch of the tile
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cc = static_cast<int>(p.chunk_count);
  int it = 0;
  int prev_series = 0, prev_chunk = 0;
  for (int series = blockIdx.x; series < p.nseries; series += gridDim.x) {
    const int64_t run = series / 6;
    const int ch = series - static_cast<int>(run) * 6;
    const int ax = ch % 3;
    const TriadNoise& e = (ch < 3) ? g.accel : g.gyro;
    const double* ref = (ch < 3) ? g.ref_accel : g.ref_gyro;
    const int64_t grun = g.run_offset + run;
    const uint32_t run_lo = static_cast<uint32_t>(grun), run_hi = static_cast<uint32_t>(grun >> 32);
    const double a = e.gm_a[ax], bgm = e.gm_b[ax], wd = e.wd[ax], wn = e.w[ax], bias = e.b[ax];
    double apow[kGenPer + 1];                              // a^q
    apow[0] = 1.0;
#pragma unroll
    for (int q = 1; q <= kGenPer; ++q) apow[q] = apow[q - 1] * a;
    double carry[1] = {0.0};                               // d at the first sample of the tile; d[0] = 0
    for (int chunk = 0; chunk < cc; ++chunk, ++it) {
      double* in = in_buf + (it & 1) * kAllanRawLen;
      const int64_t c0 = static_cast<int64_t>(chunk) * kAllanChunk;
      const int64_t left_in_series = p.len - c0;
      const int cnt = left_in_series < kAllanChunk ? static_cast<int>(left_in_series) : kAllanChunk;
      // ---- generate: white part and the zero-state drift response of this thread's stretch ------
      double mm[kGenPer], rr[kGenPer];
      double A = 1.0, E = 0.0;
      if (tid < kGenThreads) {
        double r = 0.0;
#pragma unroll
        for (int q = 0; q < kGenPer; ++q) {
          const int el = tid * kGenPer + q;
          rr[q] = r;
          mm[q] = 0.0;
          if (el < cnt) {
            const int64_t t = c0 + el;
            const Normal2 z = normal_pair(static_cast<uint32_t>(t), static_cast<uint32_t>(ch), run_lo, run_hi,
                                          g.k0, g.k1);
            mm[q] = ((ref[t * 3 + ax] + bias) + wn * z.z1) + wd * z.z0;
            r = fma(a, r, bgm * z.z0);
            A *= a;
          }
        }
        E = r;
      }
      // ---- affine scan over the threads (K1's, common.cuh) --------------------------------------
      double sA[1] = {A}, sE[1] = {E};
      affine_scan_warp<1, kAllanFastWarps>(sA, sE, wtot, lane, warp);
      __syncthreads();                                     // (1) warp totals; everybody is done with tile it-1
      if (it > 0 && tid < 9) allan_tile_fold(p, prev_series, prev_chunk, red[(it - 1) & 1]);
      double S[1];                                         // drift at the first sample of the stretch
      affine_scan_block<1, kAllanFastWarps>(sA, sE, wtot, lane, warp, carry, S);
      if (tid < kGenThreads) {
#pragma unroll
        for (int q = 0; q < kGenPer; ++q)
          in[kAllanLead + tid * kGenPer + q] = mm[q] + fma(apow[q], S[0], rr[q]);
      }
      // halo: the nine samples before the chunk are the tail of the previous tile of this series
      if (chunk != 0 && tid >= kAllanFastThreads - 9) {
        const int k = tid - (kAllanFastThreads - 9);       // 0..8 -> elements -9..-1
        const double* pin = in_buf + ((it - 1) & 1) * kAllanRawLen;
        in[1 + k] = pin[kAllanLead + kAllanChunk - 9 + k];
      }
      __syncthreads();                                     // (2) the raw tile is complete
      double* pad = pad_buf + (it & 1) * kAllanPadLen + kAllanPadLead;
      {
        const double2* in2 = reinterpret_cast<const double2*>(in);
        double2* pad2 = reinterpret_cast<double2*>(pad);
#pragma unroll
        for (int q = 0; q < 5; ++q) {
          const int u = tid + q * kAllanFastThreads;
          if (u < (kAllanLead + kAllanChunk) / 2) {
            const int ue = u - kAllanLead / 2;
            pad2[ue >= 0 ? ue + ue / 24 : ue - 1] = in2[u];
          }
        }
      }
      __syncthreads();                                     // (3) X's padded copy is complete
      double acc[4];
      if (static_cast<int64_t>(chunk + 1) * kAllanChunk <= p.len)
        allan_tile_compute<false, false>(p, series, chunk, in, pad, 0.0, acc);
      else
        allan_tile_compute<false, true>(p, series, chunk, in, pad, 0.0, acc);
      allan_tile_reduce(acc, red[it & 1]);
      prev_series = series;
      prev_chunk = chunk;
    }
  }
  __syncthreads();
  if (it > 0 && tid < 9) allan_tile_fold(p, prev_series, prev_chunk, red[(it - 1) & 1]);
}

struct AllanFinalParams {
  int64_t nseries;
  int ntau;
  double ts;
  double* avar;  // [nseries][ntau]
  double* tau;   // [ntau]
  const double* partial[kAllanMaxLevels];
  int64_t chunks[kAllanMaxLevels];
  int64_t m[128];       // cluster sizes
  int64_t nbins[128];   // floor(n / m)
  int level_of[128];
  int j_of[128];
};

// One warp per (series, tau): lane l adds the partials of chunks l, l+32, ... in order, then a
// fixed butterfly -- deterministic, and the chunk partials are read with 32 requests in flight
// instead of one dependent chain.
__global__ void __launch_bounds__(128) allan_final_kernel(const __grid_constant__ AllanFinalParams p) {
  const int64_t idx = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (idx >= p.nseries * p.ntau) return;
  const int lane = threadIdx.x & 31;
  const int64_t series = idx / p.ntau;
  const int i = static_cast<int>(idx % p.ntau);
  const int k = p.level_of[i], j = p.j_of[i];
  const double* part = p.partial[k] + series * p.chunks[k] * 9 + (j - 1);
  double s = 0.0;
  for (int64_t c = lane; c < p.chunks[k]; c += 32) s += part[c * 9];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) {
    const double m = static_cast<double>(p.m[i]);
    // avar = 0.5/(nbins-1) * sum (mean[b+1]-mean[b])^2, allan.py:54-57
    p.avar[series * p.ntau + i] = 0.5 / static_cast<double>(p.nbins[i] - 1) * (s / (m * m));
    if (series == 0) p.tau[i] = m * p.ts;  // allan.py:58
  }
}

// ---- the short upper levels in one launch ---------------------------------------------------
// Once a level has at most one chunk, it and every level above it fit in shared memory: one CTA
// per series keeps the decade sums on chip and walks the remaining levels (direct evaluation:
// one successive-difference term per thread and step), instead of one launch per level.
constexpr int kAllanRestThreads = 512;
struct AllanRestParams {
  const double* src;     // the first of these levels: x (level0 addressing) or S_k [nseries][len]
  int64_t len, src_pitch, inner, outer_stride, sample_stride;
  int level0, levels;    // number of levels handled here
  int jmax[kAllanMaxLevels];
  double* partial[kAllanMaxLevels];   // [nseries][1][9] each
};

__global__ void __launch_bounds__(kAllanRestThreads) allan_rest_kernel(const __grid_constant__ AllanRestParams p) {
  __shared__ double buf_a[kAllanChunk];        // levels k, k+2, ...
  __shared__ double buf_b[kAllanChunk / 10];   // levels k+1, k+3, ...
  __shared__ double red[kAllanRestThreads / 32][9];
  const int64_t series = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int len = static_cast<int>(p.len);
  {
    const double* base;
    int64_t stride;
    if (p.level0) {
      base = p.src + (series / p.inner) * p.outer_stride + (series % p.inner);
      stride = p.sample_stride;
    } else {
      base = p.src + series * p.src_pitch;
      stride = 1;
    }
    constexpr int kPer = (kAllanChunk + kAllanRestThreads - 1) / kAllanRestThreads;
    double v[kPer];   // every load is issued before the first store
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int e = tid + q * kAllanRestThreads;
      v[q] = (e < len) ? base[e * stride] : 0.0;
    }
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      const int e = tid + q * kAllanRestThreads;
      if (e < len) buf_a[e] = v[q];
    }
  }
  __syncthreads();
  for (int k = 0; k < p.levels; ++k) {
    const double* x = (k & 1) ? buf_b : buf_a;
    double* nx = (k & 1) ? buf_a : buf_b;
    // the first element cancels in every difference: subtracting it keeps the cluster sums small
    const double off = isfinite(x[0]) ? x[0] : 0.0;
    double acc[9];
#pragma unroll
    for (int j = 1; j <= 9; ++j) {
      double a = 0.0;
      const int nb = len / j;
      for (int b = tid; b + 1 < nb; b += kAllanRestThreads) {
        const double* q = x + b * j;
        double s0 = 0.0, s1 = 0.0;
#pragma unroll
        for (int e = 0; e < j; ++e) {
          s0 += q[e] - off;
          s1 += q[j + e] - off;
        }
        const double d = s1 - s0;
        a = fma(d, d, a);
      }
      acc[j - 1] = a;
    }
    const int nlen = len / 10;
    if (k + 1 < p.levels) {
      for (int i = tid; i < nlen; i += kAllanRestThreads) {
        const double* q = x + i * 10;
        double s0 = 0.0;
#pragma unroll
        for (int e = 0; e < 10; ++e) s0 += q[e];
        nx[i] = s0;
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
      for (int w = 0; w < kAllanRestThreads / 32; ++w) v += red[w][tid];
      p.partial[k][series * 9 + tid] = (tid < p.jmax[k]) ? v : 0.0;
    }
    __syncthreads();
    len = nlen;
  }
}

inline int64_t allan_workspace_bytes(int64_t n, int64_t nseries) {
  if (n <= 0 || nseries <= 0) return 16;
  int64_t doubles = 0;
  const int64_t n1 = (n / 10 + 2) & ~int64_t(1);   // even row pitch
  doubles += 2 * n1 * nseries;  // ping-pong decade sums
  int64_t len = n;
  for (int k = 0; k < kAllanMaxLevels && len > 0; ++k) {
    doubles += ((len + kAllanChunk - 1) / kAllanChunk) * 9 * nseries;
    len /= 10;
  }
  return doubles * static_cast<int64_t>(sizeof(double)) + 256;
}

// returns 0 on success
// gen != nullptr: level 0 is generated on the fly (allan_gen_kernel; x is not read)
inline int allan_launch(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner,
                        int64_t outer_stride, int64_t sample_stride, const int64_t* mult, int ntau,
                        double* avar, double* tau, void* workspace, int sms, cudaStream_t s,
                        const AllanGenParams* gen = nullptr) {
  AllanFinalParams fp;
  std::memset(&fp, 0, sizeof(fp));
  fp.nseries = nseries;
  fp.ntau = ntau;
  fp.ts = 1.0 / fs;
  fp.avar = avar;
  fp.tau = tau;
  int levels = 0;
  int jmax[kAllanMaxLevels] = {0};
  {
    int64_t scale = 1;
    int i = 0;
    for (int k = 0; k < kAllanMaxLevels && i < ntau; ++k, scale *= 10) {
      while (i < ntau && mult[i] / scale >= 1 && mult[i] / scale <= 9 && mult[i] % scale == 0) {
        fp.m[i] = mult[i];
        fp.nbins[i] = n / mult[i];
        fp.level_of[i] = k;
        fp.j_of[i] = static_cast<int>(mult[i] / scale);
        jmax[k] = fp.j_of[i];
        ++i;
      }
      levels = k + 1;
    }
    if (i != ntau) return 1;
  }
  double* ws = static_cast<double*>(workspace);
  const int64_t n1 = (n / 10 + 2) & ~int64_t(1);   // even row pitch: rows stay 16-byte aligned
  double* buf[2] = {ws, ws + n1 * nseries};
  double* part = ws + 2 * n1 * nseries;
  int64_t len = n;
  const size_t smem_full = (kAllanRawLen + kAllanPadLen) * sizeof(double);
  const size_t smem_stream = (kAllanStages * kAllanRawLen + 2 * kAllanPadLen) * sizeof(double);
  const size_t smem_gen = (2 * kAllanRawLen + 2 * kAllanPadLen) * sizeof(double);
  if (gen && n <= kAllanChunk) return 5;   // short series: the caller materialises them
  // function attributes are per device: remember which devices have them
  static bool attr_done[64] = {false};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
  bool& attr_set = attr_done[dev];
  if (!attr_set) {
    if (cudaFuncSetAttribute(allan_full_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             static_cast<int>(smem_full)) != cudaSuccess ||
        cudaFuncSetAttribute(allan_full_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             static_cast<int>(smem_full)) != cudaSuccess ||
        cudaFuncSetAttribute(allan_stream_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             static_cast<int>(smem_stream)) != cudaSuccess ||
        cudaFuncSetAttribute(allan_stream_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             static_cast<int>(smem_stream)) != cudaSuccess ||
        cudaFuncSetAttribute(allan_gen_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             static_cast<int>(smem_gen)) != cudaSuccess)
      return 2;
    // the kernel stages everything through shared memory: ask for the largest carve-out so that
    // two CTAs are resident per SM
    cudaFuncSetAttribute(allan_full_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    cudaFuncSetAttribute(allan_full_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    attr_set = true;
  }
  for (int k = 0; k < levels; ++k) {
    AllanLevelParams lp;
    lp.len = len;
    lp.next_len = (k + 1 < levels) ? len / 10 : 0;
    lp.nseries = nseries;
    lp.level0 = (k == 0);
    lp.src = (k == 0) ? x : buf[(k - 1) & 1];
    lp.inner = inner;
    lp.outer_stride = outer_stride;
    lp.sample_stride = sample_stride;
    lp.next = buf[k & 1];
    lp.chunks = (len + kAllanChunk - 1) / kAllanChunk;
    lp.partial = part;
    lp.jmax = jmax[k];
    lp.src_pitch = n1;
    lp.next_pitch = n1;
    fp.partial[k] = part;
    fp.chunks[k] = lp.chunks;
    part += lp.chunks * 9 * nseries;
    if (lp.chunks * nseries >= (int64_t(1) << 31)) return 4;
    if (len <= kAllanChunk) {   // this level and all above it: one launch, decade sums stay on chip
      AllanRestParams rp;
      std::memset(&rp, 0, sizeof(rp));
      rp.src = lp.src;
      rp.len = len;
      rp.src_pitch = n1;
      rp.inner = inner;
      rp.outer_stride = outer_stride;
      rp.sample_stride = sample_stride;
      rp.level0 = lp.level0;
      rp.levels = levels - k;
      int64_t l2 = len;
      for (int kk = k; kk < levels; ++kk, l2 /= 10) {
        rp.jmax[kk - k] = jmax[kk];
        rp.partial[kk - k] = part - lp.chunks * 9 * nseries + (kk - k) * 9 * nseries;
        fp.partial[kk] = rp.partial[kk - k];
        fp.chunks[kk] = 1;
      }
      allan_rest_kernel<<<static_cast<unsigned>(nseries), kAllanRestThreads, 0, s>>>(rp);
      break;
    }
    const bool contiguous = !lp.level0 || sample_stride == 1;
    // the bulk copies need 16-byte aligned rows: always true for the decade sums (even pitch),
    // for the caller's series if the base and the row stride allow it
    const bool aligned = lp.level0 ? (inner == 1 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
                                      (outer_stride & 1) == 0)
                                   : (reinterpret_cast<uintptr_t>(workspace) & 15) == 0;
    if (lp.level0 && gen) {
      // the generator front end: persistent CTAs own whole series
      lp.chunk_first = 0;
      lp.chunk_count = lp.chunks;
      const int64_t grid = nseries < sms ? nseries : sms;
      allan_gen_kernel<<<static_cast<unsigned>(grid), kAllanFastThreads, smem_gen, s>>>(lp, *gen);
    } else if (contiguous && aligned) {
      // persistent kernel, every chunk of every series (the ragged last one is masked)
      lp.chunk_first = 0;
      lp.chunk_count = lp.chunks;
      const int64_t tiles = lp.chunks * nseries;
      const int64_t grid = tiles < sms ? tiles : sms;
      if (lp.level0)
        allan_stream_kernel<false><<<static_cast<unsigned>(grid), kAllanFastThreads, smem_stream, s>>>(lp);
      else
        allan_stream_kernel<true><<<static_cast<unsigned>(grid), kAllanFastThreads, smem_stream, s>>>(lp);
    } else {
      // one tile per CTA, every chunk of every series (the ragged last one is masked)
      lp.chunk_first = 0;
      lp.chunk_count = lp.chunks;
      const int64_t tiles = lp.chunks * nseries;
      if (contiguous)
        allan_full_kernel<true><<<static_cast<unsigned>(tiles), kAllanFastThreads, smem_full, s>>>(lp);
      else
        allan_full_kernel<false><<<static_cast<unsigned>(tiles), kAllanFastThreads, smem_full, s>>>(lp);
    }
    len /= 10;
  }
  const int64_t total = nseries * ntau;
  allan_final_kernel<<<static_cast<unsigned>((total + 3) / 4), 128, 0, s>>>(fp);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

}  // namespace b2ins
