// Measures the FP64 FMA issue rate of the device (the co-roofline of the b2ins kernels,
// which are FP64-instruction-bound rather than HBM-bound) and the cost of the double
// precision libm calls the kernels lean on.   nvcc -gencode arch=compute_90a,code=sm_90a
// -O3 -o fp64_peak fp64_peak.cu && ./fp64_peak
#include <cstdio>
#include <cuda_runtime.h>

__global__ void dfma_kernel(double* out, int iters) {
  double a0 = threadIdx.x * 1e-9, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4, a5 = a0 + 5,
         a6 = a0 + 6, a7 = a0 + 7;
  const double m = 1.0000001, c = 1e-9;
  for (int i = 0; i < iters; ++i) {
    a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
    a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

template <int OP>
__global__ void libm_kernel(double* out, int iters) {
  double x = 0.3 + threadIdx.x * 1e-3, acc = 0.0;
  for (int i = 0; i < iters; ++i) {
    if (OP == 0) { double s, c; sincos(x, &s, &c); acc += s * c; }
    if (OP == 1) { acc += log(x + 1.5); }
    if (OP == 2) { double s, c; sincospi(x, &s, &c); acc += s * c; }
    if (OP == 3) { acc += sqrt(x + 2.0); }
    if (OP == 4) { acc += 1.0 / (x + 2.0); }
    x += 1e-3;
    if (x > 3.0) x -= 2.9;
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

template <typename F>
float time_ms(F f) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  f(); cudaDeviceSynchronize();
  cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); return ms;
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  const int blocks = p.multiProcessorCount * 8, threads = 256;
  double* out; cudaMalloc(&out, sizeof(double) * blocks * threads);
  const int iters = 20000;
  float ms = time_ms([&] { dfma_kernel<<<blocks, threads>>>(out, iters); });
  double fma = double(blocks) * threads * iters * 8;
  printf("{\"device\": \"%s\", \"sms\": %d, \"dfma_per_s\": %.4e, \"fp64_tflops\": %.2f, ", p.name,
         p.multiProcessorCount, fma / (ms * 1e-3), 2 * fma / (ms * 1e-3) / 1e12);
  const char* names[5] = {"sincos", "log", "sincospi", "sqrt", "rcp"};
  const int it2 = 2000;
  for (int op = 0; op < 5; ++op) {
    float t;
    if (op == 0) t = time_ms([&] { libm_kernel<0><<<blocks, threads>>>(out, it2); });
    if (op == 1) t = time_ms([&] { libm_kernel<1><<<blocks, threads>>>(out, it2); });
    if (op == 2) t = time_ms([&] { libm_kernel<2><<<blocks, threads>>>(out, it2); });
    if (op == 3) t = time_ms([&] { libm_kernel<3><<<blocks, threads>>>(out, it2); });
    if (op == 4) t = time_ms([&] { libm_kernel<4><<<blocks, threads>>>(out, it2); });
    printf("\"%s_per_s\": %.4e%s", names[op], double(blocks) * threads * it2 / (t * 1e-3),
           op == 4 ? "}\n" : ", ");
  }
  return 0;
}
