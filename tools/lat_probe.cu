// Dependent-issue latencies (cycles) of the instructions on the strapdown critical path,
// one warp on one SM.   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o lat_probe lat_probe.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int OP>
__global__ void lat(double* out, long long* cyc, int iters, double seed) {
  double x = seed + threadIdx.x * 1e-9, y = 1.0000001;
  long long t0 = clock64();
  for (int i = 0; i < iters; ++i) {
    if (OP == 0) x = fma(x, y, 1e-9);                                    // DFMA
    if (OP == 1) x = x + y;                                              // DADD
    if (OP == 2) x = 1.0 / x + 0.5;                                      // division
    if (OP == 3) x = __shfl_sync(0xffffffffu, x, (threadIdx.x + 1) & 31); // SHFL (2 per double)
    if (OP == 4) x = sqrt(x + 2.0);
    if (OP == 5) { double s, c; sincos(x, &s, &c); x = s + c; }
    if (OP == 6) x = (x > 1.5) ? x - y : x + y;                          // DSETP + select
    if (OP == 7) x = __longlong_as_double(__double_as_longlong(x) ^ 1LL) * y;  // int op + DMUL
  }
  long long t1 = clock64();
  out[threadIdx.x] = x;
  if (threadIdx.x == 0) *cyc = t1 - t0;
}

int main() {
  double* out; long long* cyc; cudaMalloc(&out, 256); cudaMalloc(&cyc, 8);
  const char* names[8] = {"dfma", "dadd", "div+add", "shfl64", "sqrt+add", "sincos+add", "dsetp+sel+dadd", "xor+dmul"};
  const int iters = 4096;
  printf("{");
  for (int op = 0; op < 8; ++op) {
    for (int rep = 0; rep < 2; ++rep) {
      switch (op) {
        case 0: lat<0><<<1, 32>>>(out, cyc, iters, 0.3); break;
        case 1: lat<1><<<1, 32>>>(out, cyc, iters, 0.3); break;
        case 2: lat<2><<<1, 32>>>(out, cyc, iters, 0.3); break;
        case 3: lat<3><<<1, 32>>>(out, cyc, iters, 0.3); break;
        case 4: lat<4><<<1, 32>>>(out, cyc, iters, 0.3); break;
        case 5: lat<5><<<1, 32>>>(out, cyc, iters, 0.3); break;
        case 6: lat<6><<<1, 32>>>(out, cyc, iters, 0.3); break;
        case 7: lat<7><<<1, 32>>>(out, cyc, iters, 0.3); break;
      }
      cudaDeviceSynchronize();
    }
    long long c; cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    printf("\"%s_cycles\": %.1f%s", names[op], double(c) / iters, op == 7 ? "}\n" : ", ");
  }
  return 0;
}
