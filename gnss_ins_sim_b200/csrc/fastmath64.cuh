// Lean double-precision elementary functions for the b2ins kernels.
//
// The Monte-Carlo kernels are bound by FP64 instruction issue, and most of those
// instructions are inside sincos / log / sincospi.  The CUDA libm versions are written for
// the whole double range (huge-argument Payne-Hanek path, denormals, NaN/Inf plumbing,
// table lookups).  Here every call site has a small, known argument range:
//   sincos_bounded   |x| <= 1e6           (Euler angles live in [-pi, pi]; lat/lon too; mech.cuh's
//                                          sincos_angle maps larger angles to 0)
//   sincospi_2u      x = 2u, u in [0, 1)  (Box-Muller angle)
//   log_unit         x in [2^-52, 1]      (Box-Muller radius)
// so a three-term Cody-Waite reduction and the classic minimax kernels (the public
// fdlibm / SunPro polynomial coefficients for sin, cos on [-pi/4, pi/4] and log on
// [sqrt(1/2), sqrt(2)]) are enough; the parity tests see ~1e-12 end to end, as with CUDA libm.
//
// Accuracy, measured on the device (H100) against an exact reference at the hard cases and ~2^22 random
// arguments per domain (tests/test_gpu_fastmath.py; the host forms in tests/test_cpu_fastmath.py):
//   sincos_bounded   |x| <= 64: <= 1.6 ulp + |q| 8.5e-32 absolute (worst 1.554 ulp), q = rint(x 2/pi):
//                    the split of pi/2 ends at PIO2_3, so results near the zeros of sin and cos, where
//                    the reduced argument is tiny, carry up to 2.6e4 ulp (3e-30 absolute);
//                    64 < |x| <= 1e6: <= 2.5 ulp + |q| 8.5e-32 (worst 2.39 ulp)
//   sincospi_2u      <= 3e-16 absolute (worst 1.94e-16); exact at 0, 1/2, 1, 3/2
//   log_unit         <= 2 ulp (worst 0.744 ulp; nvcc contracts five multiply/add pairs into DFMAs, so the
//                    device's instruction sequence is not the host's)
//   sqrt_nr          <= 0.5005 ulp on [0, 72.1] (worst 0.5: correctly rounded on every tested argument)
//   rsqrt_nr         <= 1 ulp on [0.9933, 1] (worst 0.626)
//   rcp_nr, div_nr   <= 1 ulp at their call sites (worst 0.5: correctly rounded on every tested argument)
// sincos_bounded and sincospi_2u have no contractible pairs: device and host results are identical bits.
//
// All functions are __host__ __device__ so that the accuracy check runs on the CPU.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#ifndef __CUDACC__
#define B2_HD inline
#else
#define B2_HD __host__ __device__ __forceinline__
#endif

namespace b2ins {

B2_HD double b2_fma(double a, double b, double c) {
#ifdef __CUDA_ARCH__
  return __fma_rn(a, b, c);
#else
  return std::fma(a, b, c);
#endif
}

B2_HD int32_t b2_lo32(double x) {
#ifdef __CUDA_ARCH__
  return __double2loint(x);
#else
  uint64_t u;
  std::memcpy(&u, &x, 8);
  return static_cast<int32_t>(u & 0xffffffffu);
#endif
}
B2_HD int32_t b2_hi32(double x) {
#ifdef __CUDA_ARCH__
  return __double2hiint(x);
#else
  uint64_t u;
  std::memcpy(&u, &x, 8);
  return static_cast<int32_t>(u >> 32);
#endif
}
B2_HD double b2_make(int32_t hi, int32_t lo) {
#ifdef __CUDA_ARCH__
  return __hiloint2double(hi, lo);
#else
  uint64_t u = (static_cast<uint64_t>(static_cast<uint32_t>(hi)) << 32) | static_cast<uint32_t>(lo);
  double x;
  std::memcpy(&x, &u, 8);
  return x;
#endif
}

// Constants live in __constant__ memory on the device so that they are encoded as constant-bank
// operands of DFMA/DMUL (c[3][off]) instead of being re-materialised with UMOV pairs inside
// the time loop (the profile of the first build spent a fifth of its issue slots on UMOV).
#ifdef __CUDACC__
static __constant__ double kB2Const[28] = {
    1.58969099521155010221e-10,
    -2.50507602534068634195e-08,
    2.75573137070700676789e-06,
    -1.98412698298579493134e-04,
    8.33333333332248946124e-03,
    -1.66666666666666324348e-01,
    -1.13596475577881948265e-11,
    2.08757232129817482790e-09,
    -2.75573143513906633035e-07,
    2.48015872894767294178e-05,
    -1.38888888888741095749e-03,
    4.16666666666666019037e-02,
    6.36619772367581382433e-01,
    1.57079632673412561417e+00,
    6.07710050630396597660e-11,
    2.02226624871116645580e-21,
    3.14159265358979311600e+00,
    1.22464679914735317723e-16,
    6.93147180369123816490e-01,
    1.90821492927058770002e-10,
    1.531383769920937332e-01,
    2.222219843214978396e-01,
    3.999999999940941908e-01,
    1.479819860511658591e-01,
    1.818357216161805012e-01,
    2.857142874366239149e-01,
    6.666666666666735130e-01,
    6755399441055744.0
};
#endif
#ifdef __CUDA_ARCH__
#define B2K(i, lit) (kB2Const[i])
#else
#define B2K(i, lit) (lit)
#endif

// Branch-free reciprocal, division and square root.  The IEEE-correct CUDA versions end in a
// rarely-taken slow-path CALL, which splits the basic block and stops ptxas from interleaving
// independent dependency chains (six Box-Muller pairs; the strapdown step).  These use the
// hardware seed (MUFU.RCP64H / RSQ64H, ~20 good bits) and Newton steps; results are within
// 1 ulp for normal arguments, which is all the call sites ever see.
B2_HD double rcp_nr(double x) {
#ifdef __CUDA_ARCH__
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  double e = b2_fma(-x, y, 1.0);
  y = b2_fma(y, e, y);
  e = b2_fma(-x, y, 1.0);
  y = b2_fma(y, e, y);
  return y;
#else
  return 1.0 / x;
#endif
}

// a / b, one ulp: q = a*y, then one residual correction.  The correction is itself quadratic in the error
// of y, so ONE Newton step on the hardware seed (2^-22 -> 2^-44) is enough here.
B2_HD double div_nr(double a, double b) {
#ifdef __CUDA_ARCH__
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(b));
  y = b2_fma(y, b2_fma(-b, y, 1.0), y);
  const double q = a * y;
  const double r = b2_fma(-b, q, a);
  return b2_fma(r, y, q);
#else
  return a / b;
#endif
}

// sqrt(x) for x >= 0 (x == 0 handled by a select)
B2_HD double sqrt_nr(double x) {
#ifdef __CUDA_ARCH__
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  // y ~ 1/sqrt(x): one Newton step on y (2^-22 -> 2^-43), then s = x*y with one residual correction
  // (a Heron step: quadratic again, 2^-86 before the final rounding)
  const double h = 0.5 * x;
  const double e = b2_fma(-h * y, y, 0.5);
  y = b2_fma(y, e, y);
  double s = x * y;
  const double r = b2_fma(-s, s, x);
  s = b2_fma(0.5 * r, y, s);
  return x > 0.0 ? s : 0.0;
#else
  return std::sqrt(x);
#endif
}

// 1/sqrt(x) for normal x > 0: hardware seed + two Newton steps (within 1 ulp)
B2_HD double rsqrt_nr(double x) {
#ifdef __CUDA_ARCH__
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  const double h = 0.5 * x;
  double e = b2_fma(-h * y, y, 0.5);
  y = b2_fma(y, e, y);
  e = b2_fma(-h * y, y, 0.5);
  y = b2_fma(y, e, y);
  return y;
#else
  return 1.0 / std::sqrt(x);
#endif
}

// sin and cos of r, |r| <= pi/4 (+ a little): fdlibm __kernel_sin / __kernel_cos polynomials
B2_HD void sincos_kernel(double r, double* s, double* c) {
  const double z = r * r;
  // sin: r + r z (S1 + z (S2 + z (S3 + z (S4 + z (S5 + z S6)))))
  double ps = b2_fma(z, B2K(0, 1.58969099521155010221e-10), B2K(1, -2.50507602534068634195e-08));
  ps = b2_fma(z, ps, B2K(2, 2.75573137070700676789e-06));
  ps = b2_fma(z, ps, B2K(3, -1.98412698298579493134e-04));
  ps = b2_fma(z, ps, B2K(4, 8.33333333332248946124e-03));
  ps = b2_fma(z, ps, B2K(5, -1.66666666666666324348e-01));
  *s = b2_fma(r * z, ps, r);
  // cos: 1 - z/2 + z^2 (C1 + z (C2 + z (C3 + z (C4 + z (C5 + z C6)))))
  double pc = b2_fma(z, B2K(6, -1.13596475577881948265e-11), B2K(7, 2.08757232129817482790e-09));
  pc = b2_fma(z, pc, B2K(8, -2.75573143513906633035e-07));
  pc = b2_fma(z, pc, B2K(9, 2.48015872894767294178e-05));
  pc = b2_fma(z, pc, B2K(10, -1.38888888888741095749e-03));
  pc = b2_fma(z, pc, B2K(11, 4.16666666666666019037e-02));
  // two roundings near 1 (fdlibm folds the rounding error of 1 - z/2 back for < 1 ulp; this is <= 1 ulp
  // and five operations shorter)
  *c = b2_fma(z * z, pc, b2_fma(-0.5, z, 1.0));
}

B2_HD void quadrant_fix(int q, double sr, double cr, double* s, double* c) {
  // q mod 4: 0 (s,c)  1 (c,-s)  2 (-s,-c)  3 (-c,s)
  const bool swap = q & 1;
  double ss = swap ? cr : sr;
  double cc = swap ? sr : cr;
  if (q & 2) ss = -ss;
  if ((q + 1) & 2) cc = -cc;
  *s = ss;
  *c = cc;
}

// sin(x), cos(x) for |x| <= 64 (three-term Cody-Waite: q*PIO2_1 and q*PIO2_2 are exact for |q| < 2^20)
B2_HD void sincos_bounded(double x, double* s, double* c) {
  const double kTwoOverPi = B2K(12, 6.36619772367581382433e-01);
  const double kMagic = B2K(27, 6755399441055744.0);  // 1.5 * 2^52: round-to-nearest-integer trick
  const double PIO2_1 = B2K(13, 1.57079632673412561417e+00);   // first 33 bits of pi/2
  const double PIO2_2 = B2K(14, 6.07710050630396597660e-11);   // next 33 bits
  const double PIO2_3 = B2K(15, 2.02226624871116645580e-21);   // pi/2 - (PIO2_1 + PIO2_2), leading bits
  const double t = b2_fma(x, kTwoOverPi, kMagic);
  const int q = b2_lo32(t);
  const double qd = t - kMagic;
  double r = b2_fma(-qd, PIO2_1, x);
  r = b2_fma(-qd, PIO2_2, r);
  r = b2_fma(-qd, PIO2_3, r);
  double sr, cr;
  sincos_kernel(r, &sr, &cr);
  quadrant_fix(q, sr, cr, s, c);
}

// sin(pi x), cos(pi x) for x in [0, 2]: x - q/2 is exact, the only rounding is pi*r
B2_HD void sincospi_2u(double x, double* s, double* c) {
  const double kMagic = B2K(27, 6755399441055744.0);
  const double t = b2_fma(x, 2.0, kMagic);
  const int q = b2_lo32(t);
  const double qd = t - kMagic;
  const double r = b2_fma(-qd, 0.5, x);  // exact, |r| <= 1/4
  // pi * r rounded once: |r| <= 1/4, so the angle is off by at most 2^-53 * pi/4 (half an ulp of the
  // result at worst; a double-double product would buy that back for five more operations)
  const double PI_hi = B2K(16, 3.14159265358979311600e+00);
  const double a = r * PI_hi;
  double sr, cr;
  sincos_kernel(a, &sr, &cr);
  quadrant_fix(q, sr, cr, s, c);
}

// log(x) for normal x in (0, 2): fdlibm __ieee754_log without the special cases
B2_HD double log_unit(double x) {
  const double ln2_hi = B2K(18, 6.93147180369123816490e-01);
  const double ln2_lo = B2K(19, 1.90821492927058770002e-10);
  int32_t hx = b2_hi32(x);
  const int32_t lx = b2_lo32(x);
  int k = (hx >> 20) - 1023;
  hx &= 0x000fffff;
  const int32_t i = (hx + 0x95f64) & 0x100000;  // mantissa > sqrt(2): halve it
  const double m = b2_make(hx | (i ^ 0x3ff00000), lx);
  k += (i >> 20);
  const double f = m - 1.0;
  const double s = div_nr(f, 2.0 + f);
  const double dk = static_cast<double>(k);
  const double z = s * s;
  const double w = z * z;
  double t1 = b2_fma(w, B2K(20, 1.531383769920937332e-01), B2K(21, 2.222219843214978396e-01));
  t1 = b2_fma(w, t1, B2K(22, 3.999999999940941908e-01));
  t1 = w * t1;
  double t2 = b2_fma(w, B2K(23, 1.479819860511658591e-01), B2K(24, 1.818357216161805012e-01));
  t2 = b2_fma(w, t2, B2K(25, 2.857142874366239149e-01));
  t2 = b2_fma(w, t2, B2K(26, 6.666666666666735130e-01));
  t2 = z * t2;
  const double R = t2 + t1;
  const double hfsq = 0.5 * f * f;
  return dk * ln2_hi - ((hfsq - (s * (hfsq + R) + dk * ln2_lo)) - f);
}

}  // namespace b2ins
