// Issue rate of independent FP64 / integer chains from ONE warp per SM sub-partition: cycles per
// instruction for K independent chains (K = 1..16).  With one warp per scheduler the kernels'
// serial parts are bound by this, not by the pipe's aggregate rate.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ilp_probe ilp_probe.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int K, int OP>
__global__ void ilp(double* out, long long* cyc, int iters) {
  double x[K];
  unsigned u[K];
#pragma unroll
  for (int k = 0; k < K; ++k) { x[k] = 0.3 + k + threadIdx.x * 1e-9; u[k] = threadIdx.x * 977u + k; }
  const double y = 1.0000001;
  long long t0 = clock64();
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      if (OP == 0) x[k] = fma(x[k], y, 1e-9);
      if (OP == 1) u[k] = u[k] * 0xD2511F53u + 12345u;           // IMAD
      if (OP == 2) u[k] = __umulhi(u[k], 0xD2511F53u) ^ u[k];    // IMAD.HI + LOP3
    }
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int k = 0; k < K; ++k) s += x[k] + u[k];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}

template <int K, int OP>
double run(int warps, double* out, long long* cyc) {
  const int iters = 2048;
  for (int rep = 0; rep < 2; ++rep) { ilp<K, OP><<<1, 32 * warps>>>(out, cyc, iters); cudaDeviceSynchronize(); }
  long long c; cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
  return double(c) / iters / K;
}

int main() {
  double* out; long long* cyc; cudaMalloc(&out, 8 * 1024); cudaMalloc(&cyc, 8);
  const char* names[3] = {"dfma", "imad", "imadhi_xor"};
  for (int warps : {1, 4, 8, 16}) {
    printf("{\"warps_per_sm\": %d", warps);
    printf(", \"dfma_cycles_per_inst\": {\"k1\": %.2f, \"k2\": %.2f, \"k4\": %.2f, \"k8\": %.2f, \"k16\": %.2f}",
           run<1, 0>(warps, out, cyc), run<2, 0>(warps, out, cyc), run<4, 0>(warps, out, cyc),
           run<8, 0>(warps, out, cyc), run<16, 0>(warps, out, cyc));
    printf(", \"imad_cycles_per_inst\": {\"k1\": %.2f, \"k4\": %.2f, \"k8\": %.2f}", run<1, 1>(warps, out, cyc),
           run<4, 1>(warps, out, cyc), run<8, 1>(warps, out, cyc));
    printf(", \"imadhi_xor_cycles_per_pair\": {\"k1\": %.2f, \"k4\": %.2f, \"k8\": %.2f}}\n",
           run<1, 2>(warps, out, cyc), run<4, 2>(warps, out, cyc), run<8, 2>(warps, out, cyc));
    (void)names;
  }
  return 0;
}
