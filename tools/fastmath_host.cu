// Host build of the FP64 primitives (csrc/fastmath64.cuh, mech.cuh's sincos_angle with B2INS_HOST_TEST)
// and cuRAND's own Philox4x32-10, an implementation independent of the noise generator's, for the
// CPU-side checks of tests/test_cpu_fastmath.py.  Test tooling; not part of libb2ins.so.
//   nvcc -O2 -std=c++17 -shared -Xcompiler -fPIC -DB2INS_HOST_TEST -o libfastmath_host.so tools/fastmath_host.cu
#include "../gnss_ins_sim_b200/csrc/mech.cuh"

#define QUALIFIERS static inline __host__ __device__
#include <curand_philox4x32_x.h>

using namespace b2ins;

extern "C" {

// fn as b2ins_diag_fastmath_f64 (include/b2ins.h B2INS_FM_*); host buffers
void fastmath_host(int fn, int64_t n, const double* a, const double* b, double* out0, double* out1) {
  for (int64_t i = 0; i < n; ++i) {
    double s = 0.0, c = 0.0;
    switch (fn) {
      case 0: s = rcp_nr(a[i]); break;
      case 1: s = div_nr(a[i], b[i]); break;
      case 2: s = sqrt_nr(a[i]); break;
      case 3: s = rsqrt_nr(a[i]); break;
      case 4: sincos_bounded(a[i], &s, &c); break;
      case 5: sincos_angle(a[i], &s, &c); break;
      case 6: sincospi_2u(a[i], &s, &c); break;
      default: s = log_unit(a[i]); break;
    }
    out0[i] = s;
    if (out1) out1[i] = c;
  }
}

// curand_Philox4x32_10 on ctr_key [n][6] = (counter[4], key[2]) -> words [n][4]
void philox_curand(int64_t n, const uint32_t* ck, uint32_t* words) {
  for (int64_t i = 0; i < n; ++i) {
    const uint32_t* c = ck + 6 * i;
    const uint4 r = curand_Philox4x32_10(make_uint4(c[0], c[1], c[2], c[3]), make_uint2(c[4], c[5]));
    words[4 * i] = r.x;
    words[4 * i + 1] = r.y;
    words[4 * i + 2] = r.z;
    words[4 * i + 3] = r.w;
  }
}

}  // extern "C"
