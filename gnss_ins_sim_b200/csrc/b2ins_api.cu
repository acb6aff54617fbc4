// b2ins C ABI (include/b2ins.h): argument checking, host-side pre-digestion of the error
// models, kernel dispatch, and the *_host convenience wrappers.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <type_traits>
#include <vector>

#include "../../include/b2ins.h"
#include "allan_kernel.cuh"
#include "oallan_kernel.cuh"
#include "internal.h"
#include "noise_kernel.cuh"
#include "pathgen_host.h"
#include "psd_kernel.cuh"
#include "welch_kernel.cuh"
#include "gps_kernel.cuh"
#include "mag_kernel.cuh"
#include "magcal_kernel.cuh"
#include "ekf_kernel.cuh"
#include "stats_kernel.cuh"
#include "sensor_stats_kernel.cuh"
#include "allanfit_kernel.cuh"

#ifdef B2INS_SINGLE_TU
#define B2_RF 0
#define B2_PLAIN_NAME launch_mc_plain_rf0
#define B2_SPEC_NAME launch_mc_spec_rf0
#include "mc_plain_launch.cuh"
#include "mc_spec_launch.cuh"
#undef B2_RF
#undef B2_PLAIN_NAME
#undef B2_SPEC_NAME
#define B2_RF 1
#define B2_PLAIN_NAME launch_mc_plain_rf1
#define B2_SPEC_NAME launch_mc_spec_rf1
#include "mc_plain_launch.cuh"
#include "mc_spec_launch.cuh"
#endif

using namespace b2ins;

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#define CU_CHECK(expr)                                                                    \
  do {                                                                                    \
    cudaError_t e_ = (expr);                                                              \
    if (e_ != cudaSuccess)                                                                \
      return fail(B2INS_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, \
                  __LINE__);                                                              \
  } while (0)

#define ARG_CHECK(cond, ...) \
  do {                       \
    if (!(cond)) return fail(B2INS_ERR_ARG, __VA_ARGS__); \
  } while (0)

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// bias_drift coefficients exactly as written at pathgen.py:583-586 (a: first-order
// approximation, b: exact exponential) and the white-noise scale rw/sqrt(dt) (:496-498).
int digest_triad(const b2ins_sensor_err* e, const b2ins_vib* v, double fs, TriadNoise* out) {
  const double dt = 1.0 / fs;
  for (int c = 0; c < 3; ++c) {
    out->b[c] = e->b[c];
    if (std::isinf(e->b_corr[c])) {
      out->gm_a[c] = 0.0;
      out->gm_b[c] = 0.0;
      out->wd[c] = e->b_drift[c];
    } else {
      out->gm_a[c] = 1 - 1 / fs / e->b_corr[c];
      out->gm_b[c] = e->b_drift[c] * std::sqrt(1.0 - std::exp(-2 / (fs * e->b_corr[c])));
      out->wd[c] = 0.0;
    }
    out->w[c] = e->rw[c] / std::sqrt(dt);
  }
  out->vib_type = B2INS_VIB_NONE;
  out->series_len = 0;
  out->series = nullptr;
  out->vib_w = 0.0;
  for (int c = 0; c < 3; ++c) out->vib_amp[c] = 0.0;
  if (v && v->type != B2INS_VIB_NONE) {
    ARG_CHECK(v->type >= 1 && v->type <= 3, "vib type %d is not one of B2INS_VIB_*", v->type);
    out->vib_type = v->type;
    for (int c = 0; c < 3; ++c) out->vib_amp[c] = v->amp[c];
    out->vib_w = 2.0 * M_PI * v->freq * dt;  // np.sin(2.0*math.pi*freq*dt*k), pathgen.py:491
    if (v->type == B2INS_VIB_SERIES) {
      ARG_CHECK(v->series && v->series_len > 0, "VIB_SERIES needs series and series_len > 0");
      out->series = v->series;
      out->series_len = v->series_len;
    }
  }
  return B2INS_OK;
}

void layout_strides(int layout, int64_t runs, int64_t n, int64_t* sr, int64_t* st, int64_t* sc) {
  if (layout == B2INS_LAYOUT_RUN_MAJOR) {
    *sr = n * 3;
    *st = 3;
    *sc = 1;
  } else if (layout == B2INS_LAYOUT_CHANNEL_MAJOR) {
    *sr = n * 3;
    *st = 1;
    *sc = n;
  } else {
    *sr = 1;
    *st = 3 * runs;
    *sc = runs;
  }
}

int sm_count() {
  static int cached = 0;
  if (!cached) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;   // an H100 SXM
    if (cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
      cached = 132;
  }
  return cached;
}

// tools: B2INS_MC_SHAPE="P,WI,split" overrides the specialised shape of the chosen G ("0" = the
// single-warp form); read at every launch so that one process can sweep
bool shape_override(McShape* sh) {
  const char* e = std::getenv("B2INS_MC_SHAPE");
  if (!e || !*e) return false;
  int P = 0, WI = 0, split = 0;
  const int got = std::sscanf(e, "%d,%d,%d", &P, &WI, &split);
  if (got >= 1 && P == 0) {
    sh->spec = false;
    return true;
  }
  if (got == 3) {
    sh->P = P;
    sh->WI = WI;
    sh->split = split != 0;
    sh->spec = true;
    return true;
  }
  return false;
}

// The specialised shapes that are instantiated, by group width: four-warp CTAs (one SM sub-partition
// per warp) where the group is narrow, the paired layout (producer and integrator of a group on the
// same sub-partition) for the widest groups.
// (ref_frame 1, groups of 4 and 8 lanes: the step itself split over an attitude and a velocity warp,
// mc_av_kernel.cuh, key "6,2,0" -- on an H100 0.165 against 0.177 ms at 1000 runs, 0.146 against 0.173 at 500
// at a 700 W power limit; with the shorter attitude block and lighter producers 0.137 ms at 1000 runs and
// 0.119 ms at 500 at a 400 W limit, the fused form not measured again)
McShape default_shape(int G, int rf) {
  if (rf == 1 && (G == 4 || G == 8)) return McShape{G, 6, 2, false, true};
  switch (G) {
    case 1: return McShape{1, 6, 1, false, true};
    case 2: return McShape{2, 6, 1, false, true};
    case 4: return McShape{4, 6, 1, false, true};
    case 8: return McShape{8, 6, 1, false, true};
    case 16: return McShape{16, 1, 4, true, true};
    default: return McShape{32, 1, 4, true, true};
  }
}

// Lanes per run.  The recurrence is serial in time, so the only parallelism is across runs (and,
// for the noise, across the samples and channels the producers take).  One integrator warp needs the
// same time per step whatever the number of runs it carries -- the dependent-issue latency of a single
// warp -- so with few runs the narrowest group that still gives every SM a CTA wins: fewer replicated
// lanes, fewer producer jobs per step.  With many runs G = 1 is the throughput form, and beyond
// kSpecMaxRunsG1 runs the single-warp kernel (every warp generates and integrates, five CTAs per SM)
// overtakes the specialised one.  Measured on one H100 SXM (80 GB HBM3, 700 W power limit) with
// tools/spec2_probe.py, run-steps/s at n = 1000: ref_frame 1: 500 runs G = 8 3.4e9; 1000 runs G = 4
// 6.0e9; 2000 runs G = 2 7.5e9; 4000 runs G = 2 1.0e10; 40 000 runs G = 1 1.2e10 (single-warp form
// 1.1e10); 65 536 runs single-warp form 1.49e10 (G = 1 1.24e10).  ref_frame 0: 65 536 runs single-warp
// form 1.39e10 (G = 1 1.24e10), but 100 000 runs (config 3) G = 1 1.27e10 (single-warp form 1.25e10);
// 262 144 runs single-warp form 1.53e10 (G = 1 1.27e10).
// spec_ok: the launch can take the warp-specialised form (fused noise, end-point statistics only)
constexpr int64_t kSpecMaxRunsG1[2] = {int64_t(1) << 18, int64_t(1) << 16};   // by ref_frame

int auto_lanes(int64_t runs, bool spec_ok, int sm_override = 0) {
  const int64_t sms = sm_override > 0 ? sm_override : sm_count();
  if (spec_ok) {
    // runs per CTA of the specialised shapes: 32 / G
    if (runs <= sms * 4) return 8;
    if (runs <= sms * 8) return 4;
    if (runs <= sms * 32) return 2;
    return 1;
  }
  // supplied data / process statistics (single-warp form): about one warp per SM sub-partition
  const int64_t smsp = sms * 4;
  int g = 32;
  while (g > 1 && runs * g * 2 > smsp * 32 * 3) g >>= 1;   // warps <= 1.5 per sub-partition
  return g;
}

int launch_mc(const McParams& p, int lanes, int rf, bool fed, bool proc, cudaStream_t s) {
  if (lanes != 1 && lanes != 2 && lanes != 4 && lanes != 8 && lanes != 16 && lanes != 32)
    return fail(B2INS_ERR_ARG, "lanes_per_run must be 0,1,2,4,8,16 or 32, got %d", lanes);
  if (!fed && !proc && p.algo == 0 && !(lanes == 1 && p.runs >= kSpecMaxRunsG1[rf == 1] && !std::getenv("B2INS_MC_SHAPE"))) {
    // fused noise, end-point results (and histories): the warp-specialised form
#ifdef B2INS_PHASE_CLOCKS
    if (const char* e = std::getenv("B2INS_MC_DEBUG")) const_cast<McParams&>(p).debug = std::atoi(e);
#endif
    McShape sh = default_shape(lanes, rf);
    shape_override(&sh);
    if (sh.spec) {
      sh.G = lanes;
      const bool ok = (rf == 1) ? launch_mc_spec_rf1(p, sh, s) : launch_mc_spec_rf0(p, sh, s);
      if (!ok)
        return fail(B2INS_ERR_ARG, "no specialised kernel for lanes=%d P=%d WI=%d split=%d", sh.G, sh.P,
                    sh.WI, static_cast<int>(sh.split));
      CU_CHECK(cudaGetLastError());
      return B2INS_OK;
    }
  }
  if (rf == 1)
    launch_mc_plain_rf1(p, lanes, fed, proc, s);
  else
    launch_mc_plain_rf0(p, lanes, fed, proc, s);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

struct DevBuf {
  void* p = nullptr;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 16); }
  double* d() const { return static_cast<double*>(p); }
};

// One call of a device entry point from host memory (the *_host wrappers): a stream of its own, device copies
// of the inputs queued on it, device room for the outputs and the scratch.  run() calls the device entry on
// the stream, copies the outputs back and synchronises.  After the first failed CUDA call nothing more is
// allocated or queued and run() reports that call; every buffer and the stream are released on every exit.
class Staging {
 public:
  Staging() { note(cudaStreamCreateWithFlags(&s_, cudaStreamNonBlocking), "cudaStreamCreateWithFlags"); }
  ~Staging() {
    for (const Buf& b : bufs_) cudaFree(b.dev);
    if (s_) cudaStreamDestroy(s_);
  }
  // a device copy of the `elems` doubles at host
  const double* in(const double* host, int64_t elems) {
    const size_t bytes = static_cast<size_t>(elems) * sizeof(double);
    double* d = alloc(bytes, nullptr);
    if (d && bytes) note(cudaMemcpyAsync(d, host, bytes, cudaMemcpyHostToDevice, s_), "cudaMemcpyAsync");
    return d;
  }
  // device room for `elems` doubles, copied back to host by run() unless host is null
  double* out(double* host, int64_t elems) { return alloc(static_cast<size_t>(elems) * sizeof(double), host); }
  void* scratch(int64_t bytes) { return alloc(static_cast<size_t>(bytes), nullptr); }

  template <class DeviceCall>
  int run(DeviceCall call) {
    if (err_ != cudaSuccess) return fail(B2INS_ERR_CUDA, "%s: %s", what_, cudaGetErrorString(err_));
    const int rc = call(s_);
    if (rc != B2INS_OK) return rc;
    for (const Buf& b : bufs_)
      if (b.host && b.bytes) CU_CHECK(cudaMemcpyAsync(b.host, b.dev, b.bytes, cudaMemcpyDeviceToHost, s_));
    CU_CHECK(cudaStreamSynchronize(s_));
    return B2INS_OK;
  }

 private:
  struct Buf {
    void* dev;
    void* host;
    size_t bytes;
  };
  double* alloc(size_t bytes, void* host) {
    void* p = nullptr;
    if (err_ != cudaSuccess || !note(cudaMalloc(&p, bytes ? bytes : 16), "cudaMalloc")) return nullptr;
    bufs_.push_back({p, host, bytes});
    return static_cast<double*>(p);
  }
  bool note(cudaError_t e, const char* what) {
    if (e != cudaSuccess && err_ == cudaSuccess) {
      err_ = e;
      what_ = what;
    }
    return e == cudaSuccess;
  }
  cudaStream_t s_ = nullptr;
  cudaError_t err_ = cudaSuccess;
  const char* what_ = "";
  std::vector<Buf> bufs_;
};

// What K4, K4o and K11 check in common: the sample rate, the sizes and the addressing of the series
// (series s, sample t at x[s / inner * outer_stride + (s % inner) + t * sample_stride])
int series_check(double fs, int64_t n, int64_t nseries, int64_t inner, int64_t outer_stride, int64_t sample_stride) {
  ARG_CHECK(fs > 0.0 && n >= 0 && nseries >= 0, "bad fs/n/nseries");
  ARG_CHECK(inner >= 1 && sample_stride >= 1 && outer_stride >= 0, "bad strides");
  return B2INS_OK;
}

// elements of x from the first the series read to the last (0 without series): what a *_host wrapper stages
int64_t series_elems(int64_t n, int64_t nseries, int64_t inner, int64_t outer_stride, int64_t sample_stride) {
  if (nseries == 0) return 0;
  const int64_t outer = (nseries + inner - 1) / inner;
  return (outer - 1) * outer_stride + (inner - 1) + (n - 1) * sample_stride + 1;
}

// stream-ordered scratch: freed after the work queued on s before it, on every exit path; free() does it early
// and returns the error
struct AsyncBuf {
  cudaStream_t s;
  double* p = nullptr;
  explicit AsyncBuf(cudaStream_t st) : s(st) {}
  ~AsyncBuf() {
    if (p) cudaFreeAsync(p, s);
  }
  cudaError_t alloc(size_t bytes) { return cudaMallocAsync(&p, bytes, s); }
  cudaError_t free() {
    double* q = p;
    p = nullptr;
    return q ? cudaFreeAsync(q, s) : cudaSuccess;
  }
};

// K1's time segmentation on `sms` SMs: p.nseg, p.seg_len and p.pass1_len (0 without segments) from n, runs and
// the digested decay factors.  Few runs and a long series (the Allan configuration): split the time axis into
// segments so that every SM has work.  The Gauss-Markov state at a segment start needs the draws before it:
// pass 1 reduces every segment to its zero-state end value, a tiny serial kernel chains them, pass 0
// regenerates (counter-based Philox: nothing is stored) and writes.  Costs the noise twice, so it is only used
// when one CTA per run would leave most of the GPU idle.
void noise_plan(NoiseParams* out, int sms, bool walk = false) {
  NoiseParams& p = *out;
  int nseg = 1;
  const int64_t want_ctas = static_cast<int64_t>(sms) * 2;
  if (p.runs < want_ctas && p.n >= (int64_t(1) << 18)) {
    nseg = static_cast<int>((want_ctas + p.runs - 1) / p.runs);
    const int64_t max_seg = p.n / (int64_t(1) << 16);
    if (nseg > max_seg) nseg = static_cast<int>(max_seg);
    if (nseg < 1) nseg = 1;
  }
  p.nseg = nseg;
  p.seg_len = p.n;
  p.pass1_len = 0;
  if (nseg == 1) return;
  int64_t len = (p.n + nseg - 1) / nseg;
  len = (len + kNoiseTile - 1) / kNoiseTile * kNoiseTile;   // whole tiles per segment
  p.seg_len = len;
  p.nseg = static_cast<int>((p.n + len - 1) / len);
  // pass 1 only needs the drives that still matter at the segment end: |a|^L < 1e-20.  The rule is on |a|:
  // tau < dt gives a <= 0 (-1 at tau = dt / 2), whose drives decay as |a|^k; a = 0 keeps
  // none; |a| >= 1 never decays and needs the whole segment.
  int64_t keep = walk ? len : 1;     // a rate random walk never decays
  for (int c = 0; c < 6; ++c) {
    const double a = std::fabs((c < 3) ? p.accel.gm_a[c] : p.gyro.gm_a[c - 3]);
    if (a >= 1.0) {
      keep = len;
    } else if (a > 0.0) {
      const double need = std::ceil(std::log(1e-20) / std::log(a));
      if (need > static_cast<double>(keep)) keep = need >= static_cast<double>(len) ? len : static_cast<int64_t>(need);
    }
  }
  keep = (keep + kNoiseTile - 1) / kNoiseTile * kNoiseTile;
  p.pass1_len = keep < len ? keep : len;
}

// the IEEE Std 952 terms of the two triads for the device (K1's channel order: accel, then gyro), checked; *any
// is false when every term is zero or absent, and the _ex entry points then launch the kernels without them
int digest_terms(const b2ins_noise_terms* gyro_terms, const b2ins_noise_terms* accel_terms, double fs,
                 NoiseTerms* x, bool* any, bool* walk) {
  std::memset(x, 0, sizeof(*x));
  *any = *walk = false;
  const b2ins_noise_terms* t[2] = {accel_terms, gyro_terms};
  for (int s = 0; s < 2; ++s) {
    if (!t[s]) continue;
    for (int c = 0; c < 3; ++c) {
      ARG_CHECK(std::isfinite(t[s]->q[c]) && t[s]->q[c] >= 0.0 && std::isfinite(t[s]->k[c]) && t[s]->k[c] >= 0.0 &&
                    std::isfinite(t[s]->r[c]),
                "noise terms: q and k must be finite and >= 0, r finite");
      x->q[3 * s + c] = t[s]->q[c] * std::sqrt(12.0);
      x->k[3 * s + c] = t[s]->k[c] * std::sqrt(1.0 / fs);
      x->r[3 * s + c] = t[s]->r[c];
      *any = *any || t[s]->q[c] != 0.0 || t[s]->k[c] != 0.0 || t[s]->r[c] != 0.0;
      *walk = *walk || t[s]->k[c] != 0.0;
    }
  }
  return B2INS_OK;
}

// the run-to-run errors of the two triads for the device (accel, then gyro), checked; *any is false when both are
// null or all zero, and the _rx entry points then launch exactly what the _ex ones launch
int digest_run_err(const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, RunErrs* re, bool* any) {
  std::memset(re, 0, sizeof(*re));
  *any = false;
  const b2ins_run_err* e[2] = {accel_run, gyro_run};
  for (int s = 0; s < 2; ++s) {
    if (!e[s]) continue;
    for (int c = 0; c < 3; ++c) {
      ARG_CHECK(std::isfinite(e[s]->b[c]) && e[s]->b[c] >= 0.0 && std::isfinite(e[s]->sf[c]) && e[s]->sf[c] >= 0.0,
                "run errors: b, sf and ma must be finite and >= 0");
      for (int j = 0; j < 3; ++j)
        ARG_CHECK(std::isfinite(e[s]->ma[c][j]) && e[s]->ma[c][j] >= 0.0,
                  "run errors: b, sf and ma must be finite and >= 0");
      ARG_CHECK(e[s]->ma[c][c] == 0.0, "run errors: the diagonal of ma must be 0");
      re->s[s].b[c] = e[s]->b[c];
      re->s[s].sf[c] = e[s]->sf[c];
      *any = *any || e[s]->b[c] != 0.0 || e[s]->sf[c] != 0.0;
      for (int j = 0; j < 3; ++j) {
        re->s[s].ma[c][j] = e[s]->ma[c][j];
        *any = *any || e[s]->ma[c][j] != 0.0;
      }
    }
  }
  return B2INS_OK;
}

// The error model of a K1 or K9 call, digested for the device and checked
struct NoiseModel {
  NoiseParams p;        // n, runs, dt and the two triads; noise_plan and the entry point fill in the rest
  NoiseTerms x;
  RunErrs re;
  bool terms, walk;     // a term is non-zero; a rate random walk is (digest_terms)
  bool runerr;          // a run error is non-zero (digest_run_err)
};

// The terms and the run errors are checked whatever the size; a call with no runs or no samples returns after
// them (the caller then returns B2INS_OK) and digests no triad.
int digest_noise(double fs, int64_t runs, int64_t n, const b2ins_sensor_err* gyro_err,
                 const b2ins_sensor_err* accel_err, const b2ins_noise_terms* gyro_terms,
                 const b2ins_noise_terms* accel_terms, const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                 const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, NoiseModel* m) {
  int rc = digest_terms(gyro_terms, accel_terms, fs, &m->x, &m->terms, &m->walk);
  if (rc != B2INS_OK) return rc;
  rc = digest_run_err(gyro_run, accel_run, &m->re, &m->runerr);
  if (rc != B2INS_OK || runs == 0 || n == 0) return rc;
  ARG_CHECK(gyro_err && accel_err, "null buffer");
  NoiseParams& p = m->p;
  std::memset(&p, 0, sizeof(p));
  p.n = n;
  p.runs = runs;
  p.dt = 1.0 / fs;
  rc = digest_triad(gyro_err, vib_gyro, fs, &p.gyro);
  if (rc != B2INS_OK) return rc;
  return digest_triad(accel_err, vib_accel, fs, &p.accel);
}

// The one launch site of K1 (Params = NoiseParams, pass 0 or 1) and K9 (ErrStatsParams): the form with the
// model's terms when it has any, and with its run errors when runerr
template <class Params>
void launch_noise(const Params& P, const NoiseModel& m, bool runerr, unsigned ctas, cudaStream_t s) {
  if constexpr (std::is_same_v<Params, NoiseParams>) {
    if (m.terms && runerr)
      imu_noise_ex_rx_kernel<<<ctas, kNoiseThreads, 0, s>>>(P, m.x, m.re);
    else if (m.terms)
      imu_noise_ex_kernel<<<ctas, kNoiseThreads, 0, s>>>(P, m.x);
    else if (runerr)
      imu_noise_rx_kernel<<<ctas, kNoiseThreads, 0, s>>>(P, m.re);
    else
      imu_noise_kernel<<<ctas, kNoiseThreads, 0, s>>>(P);
  } else {
    if (m.terms && runerr)
      imu_err_stats_ex_rx_kernel<<<ctas, kNoiseThreads, 0, s>>>(P, m.x, m.re);
    else if (m.terms)
      imu_err_stats_ex_kernel<<<ctas, kNoiseThreads, 0, s>>>(P, m.x);
    else if (runerr)
      imu_err_stats_rx_kernel<<<ctas, kNoiseThreads, 0, s>>>(P, m.re);
    else
      imu_err_stats_kernel<<<ctas, kNoiseThreads, 0, s>>>(P);
  }
}

// The rest of K1's parameters and its time segmentation on this device, shared by K1 and K9, after every argument
// is checked; with segments, pass 1 and the carry chain are launched here and *scratch holds their buffers until
// the caller has queued pass 0 on s.  The terms' rate random walk is carried across the segments like the drift,
// with a = 1; the run errors have no state in time, so pass 1 runs without them.
int noise_prepare(NoiseModel* m, const double* ref_gyro, const double* ref_accel, uint64_t seed, int64_t run_offset,
                  cudaStream_t s, AsyncBuf* scratch) {
  NoiseParams& p = m->p;
  const int64_t runs = p.runs;
  p.run_offset = run_offset;
  p.k0 = static_cast<uint32_t>(seed);
  p.k1 = static_cast<uint32_t>(seed >> 32);
  p.ref_gyro = ref_gyro;
  p.ref_accel = ref_accel;
  noise_plan(&p, sm_count(), m->walk);
  if (p.nseg > 1) {
    CU_CHECK(scratch->alloc(sizeof(double) * runs * p.nseg * (m->terms ? 24 : 12)));
    p.seg_end = scratch->p;
    p.seg_carry = scratch->p + runs * p.nseg * 6;
    if (m->terms) {
      m->x.seg_end = scratch->p + runs * p.nseg * 12;
      m->x.seg_carry = scratch->p + runs * p.nseg * 18;
    }
    p.pass = 1;
    launch_noise(p, *m, false, static_cast<unsigned>(runs * (p.nseg - 1)), s);
    const unsigned ctas = static_cast<unsigned>((runs * 6 + 127) / 128);
    if (m->terms) {
      NoiseParams pw = p;      // the walk's carry chain: noise_carry_kernel with a = 1
      for (int c = 0; c < 3; ++c) pw.accel.gm_a[c] = pw.gyro.gm_a[c] = 1.0;
      pw.seg_end = m->x.seg_end;
      pw.seg_carry = m->x.seg_carry;
      noise_carry_kernel<<<ctas, 128, 0, s>>>(pw);
    }
    noise_carry_kernel<<<ctas, 128, 0, s>>>(p);
    p.pass = 0;
  }
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

}  // namespace

extern "C" {

int b2ins_version(void) { return B2INS_VERSION; }

const char* b2ins_last_error(void) { return g_err; }

int b2ins_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

// allan.py:29-44
int b2ins_allan_num_tau(int64_t n, double fs, int64_t* m, int m_cap) {
  const double ts = 1.0 / fs;
  const int64_t max_bin = static_cast<int64_t>(std::floor(n / 9.0));
  if (max_bin * ts < 1) return 0;
  const int nextpow10 = static_cast<int>(std::ceil(std::log10(static_cast<double>(max_bin))));
  int count = 0;
  double scale = 0.1;
  for (int i = 0; i < nextpow10; ++i) {
    scale *= 10;
    for (int j = 1; j < 10; ++j) {
      const int64_t tmp = static_cast<int64_t>(j * scale);
      if (tmp <= max_bin) {
        if (m && count < m_cap) m[count] = tmp;
        ++count;
      } else {
        break;
      }
    }
  }
  return count;
}

// ---------------------------------------------------------------- K2 --------
static int free_integration_fed(int algo, int ref_frame, double fs, int64_t runs, int64_t n,
                                const double* gyro, const double* accel, int layout,
                                const double* ini, int ini_sets, int ini_rows, int64_t run_offset,
                                int earth_rot, double* att, double* pos, double* vel,
                                int lanes_per_run, void* stream) {
  ARG_CHECK(ref_frame == 0 || ref_frame == 1, "ref_frame must be 0 or 1, got %d", ref_frame);
  ARG_CHECK(fs > 0.0, "fs must be positive");
  ARG_CHECK(runs >= 0 && n >= 0, "runs and n must be non-negative");
  ARG_CHECK(layout == 0 || layout == 1, "layout must be B2INS_LAYOUT_*");
  ARG_CHECK(ini_sets >= 1 && (ini_rows == 9 || ini_rows == 10), "ini must be [sets>=1][9|10]");
  if (runs == 0 || n == 0) return B2INS_OK;
  ARG_CHECK(gyro && accel && ini && att && pos && vel, "null buffer");
  ARG_CHECK(n < (int64_t(1) << 32), "n must be < 2^32");
  McParams p;
  std::memset(&p, 0, sizeof(p));
  p.n = n;
  p.runs = runs;
  p.run_offset = run_offset;
  p.ini_offset = run_offset;
  p.dt = 1.0 / fs;
  p.earth_rot = earth_rot;
  p.ini = ini;
  p.ini_sets = ini_sets;
  p.ini_rows = ini_rows;
  p.fed_gyro = gyro;
  p.fed_accel = accel;
  layout_strides(layout, runs, n, &p.sr, &p.st, &p.sc);
  p.algo = algo;
  if (algo == 1) {   // `accel` carries the odometer series [R][n] or [n][R]
    p.fed_accel = nullptr;
    p.fed_odo = accel;
    p.so_r = (layout == B2INS_LAYOUT_RUN_MAJOR) ? n : 1;
    p.so_t = (layout == B2INS_LAYOUT_RUN_MAJOR) ? 1 : runs;
  }
  p.out_att = att;
  p.out_pos = pos;
  p.out_vel = vel;
  p.osr = p.sr;
  p.ost = p.st;
  p.osc = p.sc;
  p.dump_runs = runs;
  p.dump_stride = 1;
  p.dump_rows = n;
  p.stats_start = -1;
  int lanes = lanes_per_run;
  if (lanes == 0) {
    lanes = auto_lanes(runs, false);
    // run-major rows are 24-byte strided per lane when G = 1; a wider group reads whole
    // contiguous stretches of one run
    if (layout == B2INS_LAYOUT_RUN_MAJOR && lanes < 8) lanes = 8;
  }
  return launch_mc(p, lanes, ref_frame, true, false, static_cast<cudaStream_t>(stream));
}

int b2ins_free_integration_f64(int ref_frame, double fs, int64_t runs, int64_t n,
                               const double* gyro, const double* accel, int layout,
                               const double* ini, int ini_sets, int ini_rows, int64_t run_offset,
                               int earth_rot, double* att, double* pos, double* vel,
                               int lanes_per_run, void* stream) {
  return free_integration_fed(0, ref_frame, fs, runs, n, gyro, accel, layout, ini, ini_sets,
                              ini_rows, run_offset, earth_rot, att, pos, vel, lanes_per_run, stream);
}

int b2ins_free_integration_odo_f64(int ref_frame, double fs, int64_t runs, int64_t n,
                                   const double* gyro, const double* odo, int layout,
                                   const double* ini, int ini_sets, int ini_rows,
                                   int64_t run_offset, int earth_rot, double* att, double* pos,
                                   double* vel, int lanes_per_run, void* stream) {
  return free_integration_fed(1, ref_frame, fs, runs, n, gyro, odo, layout, ini, ini_sets,
                              ini_rows, run_offset, earth_rot, att, pos, vel, lanes_per_run, stream);
}

int b2ins_free_integration_f64_host(int ref_frame, double fs, int64_t runs, int64_t n,
                                    const double* gyro, const double* accel, int layout,
                                    const double* ini, int ini_sets, int ini_rows,
                                    int64_t run_offset, int earth_rot, double* att, double* pos,
                                    double* vel, int lanes_per_run) {
  ARG_CHECK(runs >= 0 && n >= 0, "runs and n must be non-negative");
  if (runs == 0 || n == 0) return B2INS_OK;
  ARG_CHECK(gyro && accel && ini && att && pos && vel, "null buffer");
  ARG_CHECK(ini_sets >= 1 && (ini_rows == 9 || ini_rows == 10), "ini must be [sets>=1][9|10]");
  const int64_t elems = runs * n * 3;
  Staging st;
  const double* dg = st.in(gyro, elems);
  const double* da = st.in(accel, elems);
  const double* di = st.in(ini, int64_t(ini_sets) * ini_rows);
  double* oa = st.out(att, elems);
  double* op = st.out(pos, elems);
  double* ov = st.out(vel, elems);
  return st.run([&](cudaStream_t s) {
    return b2ins_free_integration_f64(ref_frame, fs, runs, n, dg, da, layout, di, ini_sets, ini_rows, run_offset,
                                      earth_rot, oa, op, ov, lanes_per_run, s);
  });
}

// ---------------------------------------------------------------- K1 --------
int b2ins_imu_noise_rx_f64(double fs, int64_t runs, int64_t n, const double* ref_gyro,
                           const double* ref_accel, const b2ins_sensor_err* gyro_err,
                           const b2ins_sensor_err* accel_err, const b2ins_noise_terms* gyro_terms,
                           const b2ins_noise_terms* accel_terms, const b2ins_vib* vib_gyro,
                           const b2ins_vib* vib_accel, uint64_t seed, int64_t run_offset, int layout,
                           double* gyro, double* accel, double* z_dump, const b2ins_run_err* gyro_run,
                           const b2ins_run_err* accel_run, void* stream) {
  ARG_CHECK(fs > 0.0, "fs must be positive");
  ARG_CHECK(runs >= 0 && n >= 0, "runs and n must be non-negative");
  ARG_CHECK(layout >= 0 && layout <= 2, "layout must be B2INS_LAYOUT_*");
  NoiseModel m;
  int rc = digest_noise(fs, runs, n, gyro_err, accel_err, gyro_terms, accel_terms, vib_gyro, vib_accel, gyro_run,
                        accel_run, &m);
  if (rc != B2INS_OK || runs == 0 || n == 0) return rc;
  ARG_CHECK(ref_gyro && ref_accel && gyro && accel, "null buffer");
  ARG_CHECK(n < (int64_t(1) << 32), "n must be < 2^32");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AsyncBuf scratch(s);
  rc = noise_prepare(&m, ref_gyro, ref_accel, seed, run_offset, s, &scratch);
  if (rc != B2INS_OK) return rc;
  NoiseParams& p = m.p;
  p.out_gyro = gyro;
  p.out_accel = accel;
  layout_strides(layout, runs, n, &p.osr, &p.ost, &p.osc);
  p.z_dump = z_dump;
  launch_noise(p, m, m.runerr, static_cast<unsigned>(runs * p.nseg), s);
  CU_CHECK(scratch.free());
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_imu_noise_ex_f64(double fs, int64_t runs, int64_t n, const double* ref_gyro,
                           const double* ref_accel, const b2ins_sensor_err* gyro_err,
                           const b2ins_sensor_err* accel_err, const b2ins_noise_terms* gyro_terms,
                           const b2ins_noise_terms* accel_terms, const b2ins_vib* vib_gyro,
                           const b2ins_vib* vib_accel, uint64_t seed, int64_t run_offset, int layout,
                           double* gyro, double* accel, double* z_dump, void* stream) {
  return b2ins_imu_noise_rx_f64(fs, runs, n, ref_gyro, ref_accel, gyro_err, accel_err, gyro_terms, accel_terms,
                                vib_gyro, vib_accel, seed, run_offset, layout, gyro, accel, z_dump, nullptr, nullptr,
                                stream);
}

int b2ins_imu_noise_f64(double fs, int64_t runs, int64_t n, const double* ref_gyro,
                        const double* ref_accel, const b2ins_sensor_err* gyro_err,
                        const b2ins_sensor_err* accel_err, const b2ins_vib* vib_gyro,
                        const b2ins_vib* vib_accel, uint64_t seed, int64_t run_offset, int layout,
                        double* gyro, double* accel, double* z_dump, void* stream) {
  return b2ins_imu_noise_ex_f64(fs, runs, n, ref_gyro, ref_accel, gyro_err, accel_err, nullptr, nullptr, vib_gyro,
                                vib_accel, seed, run_offset, layout, gyro, accel, z_dump, stream);
}

int b2ins_imu_run_err_f64(uint64_t seed, int64_t runs, int64_t run_offset, const b2ins_run_err* gyro_run,
                          const b2ins_run_err* accel_run, double* out, void* stream) {
  ARG_CHECK(runs >= 0, "runs must be non-negative");
  RunErrs re;
  bool any = false;
  const int rc = digest_run_err(gyro_run, accel_run, &re, &any);
  if (rc != B2INS_OK) return rc;
  if (runs == 0) return B2INS_OK;
  ARG_CHECK(out, "null buffer");
  imu_run_err_kernel<<<static_cast<unsigned>((runs * 2 + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      re, runs, run_offset, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32), out);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

// ---------------------------------------------------------------- K9 --------
int b2ins_imu_err_stats_rx_f64(double fs, int64_t runs, int64_t n, const double* ref_gyro, const double* ref_accel,
                               const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                               const b2ins_noise_terms* gyro_terms, const b2ins_noise_terms* accel_terms,
                               const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel, uint64_t seed,
                               int64_t run_offset, int64_t stats_start, double* end_err, double* proc_stats,
                               const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, void* stream) {
  ARG_CHECK(fs > 0.0, "fs must be positive");
  ARG_CHECK(runs >= 0 && n >= 0, "runs and n must be non-negative");
  ARG_CHECK(stats_start < n || n == 0, "stats_start must be < n");
  NoiseModel m;
  int rc = digest_noise(fs, runs, n, gyro_err, accel_err, gyro_terms, accel_terms, vib_gyro, vib_accel, gyro_run,
                        accel_run, &m);
  if (rc != B2INS_OK || runs == 0 || n == 0) return rc;
  ARG_CHECK(ref_gyro && ref_accel && end_err, "null buffer");
  ARG_CHECK(stats_start < 0 || proc_stats, "stats_start >= 0 needs proc_stats");
  ARG_CHECK(n < (int64_t(1) << 32), "n must be < 2^32");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AsyncBuf scratch(s), partial(s);
  rc = noise_prepare(&m, ref_gyro, ref_accel, seed, run_offset, s, &scratch);
  if (rc != B2INS_OK) return rc;
  ErrStatsParams P;
  std::memset(&P, 0, sizeof(P));
  P.np = m.p;
  P.stats_start = stats_start;
  P.end_err = end_err;
  P.proc_stats = proc_stats;
  if (P.np.nseg > 1 && stats_start >= 0) {
    const cudaError_t e = partial.alloc(sizeof(double) * runs * P.np.nseg * kErrPartial);
    if (e != cudaSuccess)
      return fail(B2INS_ERR_CUDA, "cudaMallocAsync of the segment partials: %s", cudaGetErrorString(e));
    P.partial = partial.p;
  }
  launch_noise(P, m, m.runerr, static_cast<unsigned>(runs * P.np.nseg), s);
  if (partial.p) {
    err_stats_fold_kernel<<<static_cast<unsigned>((runs * kErrCh + 127) / 128), 128, 0, s>>>(P);
    CU_CHECK(partial.free());
  }
  CU_CHECK(scratch.free());
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_imu_err_stats_ex_f64(double fs, int64_t runs, int64_t n, const double* ref_gyro, const double* ref_accel,
                               const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                               const b2ins_noise_terms* gyro_terms, const b2ins_noise_terms* accel_terms,
                               const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel, uint64_t seed,
                               int64_t run_offset, int64_t stats_start, double* end_err, double* proc_stats,
                               void* stream) {
  return b2ins_imu_err_stats_rx_f64(fs, runs, n, ref_gyro, ref_accel, gyro_err, accel_err, gyro_terms, accel_terms,
                                    vib_gyro, vib_accel, seed, run_offset, stats_start, end_err, proc_stats, nullptr,
                                    nullptr, stream);
}

int b2ins_imu_err_stats_f64(double fs, int64_t runs, int64_t n, const double* ref_gyro, const double* ref_accel,
                            const b2ins_sensor_err* gyro_err, const b2ins_sensor_err* accel_err,
                            const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel, uint64_t seed, int64_t run_offset,
                            int64_t stats_start, double* end_err, double* proc_stats, void* stream) {
  return b2ins_imu_err_stats_ex_f64(fs, runs, n, ref_gyro, ref_accel, gyro_err, accel_err, nullptr, nullptr, vib_gyro,
                                    vib_accel, seed, run_offset, stats_start, end_err, proc_stats, stream);
}

// ---------------------------------------------------------------- K3p -------
int b2ins_proc_stats_f64(int64_t runs, int64_t m, int ncomp, const double* x, const double* ref, int64_t start,
                         double* end_err, double* proc_stats, void* stream) {
  ARG_CHECK(runs >= 0 && m >= 0, "runs and m must be non-negative");
  ARG_CHECK(ncomp >= 1 && ncomp <= kProcMaxComp, "ncomp must be in 1..%d, got %d", kProcMaxComp, ncomp);
  ARG_CHECK(start >= 0 && (start < m || m == 0), "start must be in [0, m)");
  if (runs == 0 || m == 0) return B2INS_OK;
  ARG_CHECK(x && ref && end_err && proc_stats, "null buffer");
  ARG_CHECK(runs < (int64_t(1) << 31), "runs must be < 2^31");
  proc_stats_kernel<<<static_cast<unsigned>(runs), kProcThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      m, ncomp, x, ref, start, end_err, proc_stats);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_gps_noise_f64(int64_t runs, int64_t m, const double* ref_gps, const double* stdp,
                        const double* stdv, int gps_type, uint64_t seed, int64_t run_offset,
                        double* gps, void* stream) {
  ARG_CHECK(runs >= 0 && m >= 0, "runs and m must be non-negative");
  ARG_CHECK(gps_type == 0 || gps_type == 1, "gps_type must be 0 (LLA) or 1 (xyz)");
  if (runs == 0 || m == 0) return B2INS_OK;
  ARG_CHECK(ref_gps && stdp && stdv && gps, "null buffer");
  ARG_CHECK(m < (int64_t(1) << 32), "m must be < 2^32");
  GpsParams p;
  p.m = m;
  p.runs = runs;
  p.run_offset = run_offset;
  p.ref = ref_gps;
  p.out = gps;
  for (int i = 0; i < 3; ++i) {
    p.stdp[i] = stdp[i];
    p.stdv[i] = stdv[i];
  }
  p.k0 = static_cast<uint32_t>(seed);
  p.k1 = static_cast<uint32_t>(seed >> 32);
  p.gps_type = gps_type;
  const int64_t total = runs * m;
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  gps_noise_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_mag_noise_f64(int64_t runs, int64_t n, const double* ref_mag, const double* si,
                        const double* hi, const double* std, uint64_t seed, int64_t run_offset,
                        double* mag, void* stream) {
  ARG_CHECK(runs >= 0 && n >= 0, "runs and n must be non-negative");
  ARG_CHECK(si && hi && std, "null error model");
  for (int i = 0; i < 3; ++i)
    ARG_CHECK(std::isfinite(std[i]) && std[i] >= 0.0, "mag std must be finite and >= 0");
  if (runs == 0 || n == 0) return B2INS_OK;
  ARG_CHECK(ref_mag && mag, "null buffer");
  ARG_CHECK(n < (int64_t(1) << 32), "n must be < 2^32");
  MagParams p;
  p.n = n;
  p.runs = runs;
  p.run_offset = run_offset;
  p.ref = ref_mag;
  p.out = mag;
  for (int i = 0; i < 9; ++i) p.si[i] = si[i];
  for (int i = 0; i < 3; ++i) {
    p.hi[i] = hi[i];
    p.std[i] = std[i];
  }
  p.k0 = static_cast<uint32_t>(seed);
  p.k1 = static_cast<uint32_t>(seed >> 32);
  const int64_t total = runs * n;
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = static_cast<int64_t>(sm_count()) * 16;
  if (blocks > cap) blocks = cap;
  mag_noise_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(p);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

// ---------------------------------------------------------------- K10 -------
static int magcal_check(int64_t runs, int64_t n, const int64_t* seg, MagCalParams* p) {
  ARG_CHECK(runs >= 0 && n >= 0, "runs and n must be non-negative");
  ARG_CHECK(seg, "null segments");
  ARG_CHECK(runs < (int64_t(1) << 31), "runs must be < 2^31");
  ARG_CHECK(n < (int64_t(1) << 32), "n must be < 2^32");
  for (int i = 0; i < 3; ++i)
    ARG_CHECK(seg[2 * i] >= 0 && seg[2 * i + 1] <= n && seg[2 * i + 1] - seg[2 * i] >= 3,
              "segment %d [%lld, %lld) must hold at least 3 rows inside [0, %lld)", i, (long long)seg[2 * i],
              (long long)seg[2 * i + 1], (long long)n);
  std::memset(p, 0, sizeof(*p));
  p->runs = runs;
  p->n = n;
  for (int i = 0; i < 6; ++i) p->seg[i] = seg[i];
  return B2INS_OK;
}

int b2ins_magcal_f64(int64_t runs, int64_t n, const int64_t* seg, const double* ref_mag, const double* si,
                     const double* hi, const double* std, uint64_t seed, int64_t run_offset, double* soft_iron,
                     double* hard_iron, double* err, void* stream) {
  MagCalParams p;
  const int rc = magcal_check(runs, n, seg, &p);
  if (rc != B2INS_OK) return rc;
  ARG_CHECK(si && hi && std, "null error model");
  for (int i = 0; i < 3; ++i)
    ARG_CHECK(std::isfinite(std[i]) && std[i] >= 0.0, "mag std must be finite and >= 0");
  if (runs == 0) return B2INS_OK;
  ARG_CHECK(ref_mag && soft_iron && hard_iron, "null buffer");
  p.run_offset = run_offset;
  p.ref = ref_mag;
  for (int i = 0; i < 9; ++i) p.si[i] = si[i];
  for (int i = 0; i < 3; ++i) {
    p.hi[i] = hi[i];
    p.std[i] = std[i];
  }
  p.k0 = static_cast<uint32_t>(seed);
  p.k1 = static_cast<uint32_t>(seed >> 32);
  p.soft_iron = soft_iron;
  p.hard_iron = hard_iron;
  p.err = err;
  magcal_kernel<false><<<static_cast<unsigned>(runs), kMagCalThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_magcal_fed_f64(int64_t runs, int64_t n, const int64_t* seg, const double* mag, int64_t run_stride,
                         int64_t sample_stride, double* soft_iron, double* hard_iron, double* mag_cal,
                         void* stream) {
  MagCalParams p;
  const int rc = magcal_check(runs, n, seg, &p);
  if (rc != B2INS_OK) return rc;
  ARG_CHECK(run_stride >= 0 && sample_stride >= 3, "run_stride must be >= 0 and sample_stride >= 3");
  if (runs == 0) return B2INS_OK;
  ARG_CHECK(mag && soft_iron && hard_iron, "null buffer");
  p.x = mag;
  p.run_stride = run_stride;
  p.sample_stride = sample_stride;
  p.soft_iron = soft_iron;
  p.hard_iron = hard_iron;
  p.mag_cal = mag_cal;
  magcal_kernel<true><<<static_cast<unsigned>(runs), kMagCalThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_magcal_fed_f64_host(int64_t runs, int64_t n, const int64_t* seg, const double* mag, int64_t run_stride,
                              int64_t sample_stride, double* soft_iron, double* hard_iron, double* mag_cal) {
  MagCalParams chk;
  const int rc = magcal_check(runs, n, seg, &chk);
  if (rc != B2INS_OK) return rc;
  ARG_CHECK(run_stride >= 0 && sample_stride >= 3, "run_stride must be >= 0 and sample_stride >= 3");
  if (runs == 0) return B2INS_OK;
  ARG_CHECK(mag && soft_iron && hard_iron, "null buffer");
  const int64_t L = (seg[1] - seg[0]) + (seg[3] - seg[2]) + (seg[5] - seg[4]);
  Staging st;
  const double* dx = st.in(mag, (runs - 1) * run_stride + (n - 1) * sample_stride + 3);
  double* dsi = st.out(soft_iron, runs * 9);
  double* dhi = st.out(hard_iron, runs * 4);
  double* dcal = mag_cal ? st.out(mag_cal, runs * L * 3) : nullptr;
  return st.run([&](cudaStream_t s) {
    return b2ins_magcal_fed_f64(runs, n, seg, dx, run_stride, sample_stride, dsi, dhi, dcal, s);
  });
}

int b2ins_imu_noise_f64_host(double fs, int64_t runs, int64_t n, const double* ref_gyro,
                             const double* ref_accel, const b2ins_sensor_err* gyro_err,
                             const b2ins_sensor_err* accel_err, const b2ins_vib* vib_gyro,
                             const b2ins_vib* vib_accel, uint64_t seed, int64_t run_offset,
                             int layout, double* gyro, double* accel, double* z_dump) {
  return b2ins_imu_noise_ex_f64_host(fs, runs, n, ref_gyro, ref_accel, gyro_err, accel_err, nullptr, nullptr,
                                     vib_gyro, vib_accel, seed, run_offset, layout, gyro, accel, z_dump);
}

int b2ins_imu_noise_ex_f64_host(double fs, int64_t runs, int64_t n, const double* ref_gyro,
                                const double* ref_accel, const b2ins_sensor_err* gyro_err,
                                const b2ins_sensor_err* accel_err, const b2ins_noise_terms* gyro_terms,
                                const b2ins_noise_terms* accel_terms, const b2ins_vib* vib_gyro,
                                const b2ins_vib* vib_accel, uint64_t seed, int64_t run_offset,
                                int layout, double* gyro, double* accel, double* z_dump) {
  return b2ins_imu_noise_rx_f64_host(fs, runs, n, ref_gyro, ref_accel, gyro_err, accel_err, gyro_terms, accel_terms,
                                     vib_gyro, vib_accel, seed, run_offset, layout, gyro, accel, z_dump, nullptr,
                                     nullptr);
}

int b2ins_imu_noise_rx_f64_host(double fs, int64_t runs, int64_t n, const double* ref_gyro,
                                const double* ref_accel, const b2ins_sensor_err* gyro_err,
                                const b2ins_sensor_err* accel_err, const b2ins_noise_terms* gyro_terms,
                                const b2ins_noise_terms* accel_terms, const b2ins_vib* vib_gyro,
                                const b2ins_vib* vib_accel, uint64_t seed, int64_t run_offset,
                                int layout, double* gyro, double* accel, double* z_dump,
                                const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run) {
  ARG_CHECK(runs >= 0 && n >= 0, "runs and n must be non-negative");
  RunErrs re;
  bool runerr = false;
  const int rc = digest_run_err(gyro_run, accel_run, &re, &runerr);
  if (rc != B2INS_OK) return rc;
  if (runs == 0 || n == 0) return B2INS_OK;
  ARG_CHECK(ref_gyro && ref_accel && gyro && accel, "null buffer");
  ARG_CHECK(!(vib_gyro && vib_gyro->type == B2INS_VIB_SERIES) &&
                !(vib_accel && vib_accel->type == B2INS_VIB_SERIES),
            "VIB_SERIES takes a device pointer: use the device entry point");
  const int64_t ref = n * 3, elems = runs * ref;
  Staging st;
  const double* rg = st.in(ref_gyro, ref);
  const double* ra = st.in(ref_accel, ref);
  double* og = st.out(gyro, elems);
  double* oa = st.out(accel, elems);
  double* zd = z_dump ? st.out(z_dump, elems * 4) : nullptr;
  return st.run([&](cudaStream_t s) {
    return b2ins_imu_noise_rx_f64(fs, runs, n, rg, ra, gyro_err, accel_err, gyro_terms, accel_terms, vib_gyro,
                                  vib_accel, seed, run_offset, layout, og, oa, zd, gyro_run, accel_run, s);
  });
}

// ---------------------------------------------------------------- K12 -------
int b2ins_mc_free_integration_ex_f64(const b2ins_mc_config* cfg, int proc_pos_frame, const double* ref_gyro,
                                     const double* ref_accel, const double* ref_nav,
                                     const double* ini, double* end_err, double* end_state,
                                     double* proc_stats, double* dump_att, double* dump_pos,
                                     double* dump_vel, double* dump_gyro, double* dump_accel,
                                     void* stream) {
  ARG_CHECK(cfg, "cfg is null");
  ARG_CHECK(cfg->ref_frame == 0 || cfg->ref_frame == 1, "ref_frame must be 0 or 1");
  ARG_CHECK(proc_pos_frame >= B2INS_POS_FRAME_LLA && proc_pos_frame <= B2INS_POS_FRAME_ECEF,
            "proc_pos_frame must be B2INS_POS_FRAME_*");
  ARG_CHECK(proc_pos_frame == B2INS_POS_FRAME_LLA || cfg->ref_frame == 0,
            "proc_pos_frame NED / ECEF needs ref_frame 0 (LLA positions)");
  ARG_CHECK(cfg->fs > 0.0, "fs must be positive");
  ARG_CHECK(cfg->runs >= 0 && cfg->n >= 0, "runs and n must be non-negative");
  ARG_CHECK(cfg->ini_sets >= 1 && (cfg->ini_rows == 9 || cfg->ini_rows == 10),
            "ini must be [sets>=1][9|10]");
  if (cfg->runs == 0 || cfg->n == 0) return B2INS_OK;
  ARG_CHECK(ref_gyro && ref_accel && ini, "null input buffer");
  ARG_CHECK(aligned16(ref_gyro) && aligned16(ref_accel) && aligned16(ref_nav),
            "ref_gyro / ref_accel / ref_nav must be 16-byte aligned (bulk async copies)");
  ARG_CHECK(cfg->n < (int64_t(1) << 32), "n must be < 2^32");
  ARG_CHECK(!(end_err || cfg->stats_start >= 0) || ref_nav, "ref_nav is needed for errors");
  ARG_CHECK(cfg->stats_start < 0 || proc_stats, "stats_start >= 0 needs proc_stats");
  ARG_CHECK(cfg->dump_runs >= 0 && cfg->dump_runs <= cfg->runs, "dump_runs out of range");
  ARG_CHECK((!dump_att && !dump_pos && !dump_vel) || (dump_att && dump_pos && dump_vel),
            "dump_att/pos/vel must be given together");
  ARG_CHECK((!dump_gyro) == (!dump_accel), "dump_gyro/accel must be given together");
  McParams p;
  std::memset(&p, 0, sizeof(p));
  p.n = cfg->n;
  p.runs = cfg->runs;
  p.run_offset = cfg->run_offset;
  p.ini_offset = cfg->ini_offset;
  p.dt = 1.0 / cfg->fs;
  p.earth_rot = cfg->earth_rot;
  p.k0 = static_cast<uint32_t>(cfg->seed);
  p.k1 = static_cast<uint32_t>(cfg->seed >> 32);
  int rc = digest_triad(&cfg->gyro_err, &cfg->vib_gyro, cfg->fs, &p.gyro);
  if (rc != B2INS_OK) return rc;
  rc = digest_triad(&cfg->accel_err, &cfg->vib_accel, cfg->fs, &p.accel);
  if (rc != B2INS_OK) return rc;
  p.ref_gyro = ref_gyro;
  p.ref_accel = ref_accel;
  p.ref_nav = ref_nav;
  p.ini = ini;
  p.ini_sets = cfg->ini_sets;
  p.ini_rows = cfg->ini_rows;
  p.out_att = dump_att;
  p.out_pos = dump_pos;
  p.out_vel = dump_vel;
  p.out_gyro = dump_gyro;
  p.out_accel = dump_accel;
  ARG_CHECK(cfg->dump_stride >= 0, "dump_stride must be >= 0");
  p.dump_stride = cfg->dump_stride > 1 ? cfg->dump_stride : 1;
  p.dump_rows = (cfg->n + p.dump_stride - 1) / p.dump_stride;
  layout_strides(B2INS_LAYOUT_RUN_MAJOR, cfg->dump_runs, p.dump_rows, &p.osr, &p.ost, &p.osc);
  p.dump_runs = (dump_att || dump_gyro) ? cfg->dump_runs : 0;
  ARG_CHECK(!cfg->dump_quat || dump_att, "dump_quat needs the attitude histories (dump_att)");
  p.out_quat = cfg->dump_quat;
  p.end_err = end_err;
  p.end_state = end_state;
  p.proc_stats = proc_stats;
  p.stats_start = cfg->stats_start;
  p.proc_pos_frame = proc_pos_frame;
  ARG_CHECK(cfg->algo == 0 || cfg->algo == 1, "algo must be 0 (free integration) or 1 (odometer)");
  p.algo = cfg->algo;
  if (cfg->algo == 1) {
    ARG_CHECK(cfg->ref_odo, "algo 1 needs ref_odo");
    p.ref_odo = cfg->ref_odo;
    p.odo_scale = cfg->odo_scale;
    p.odo_stdv = cfg->odo_stdv;
    p.out_odo = cfg->dump_odo;
    if (cfg->dump_odo && p.dump_runs == 0) p.dump_runs = cfg->dump_runs;
  }
  const int lanes = cfg->lanes_per_run ? cfg->lanes_per_run : auto_lanes(cfg->runs, cfg->stats_start < 0);
  return launch_mc(p, lanes, cfg->ref_frame, false, cfg->stats_start >= 0,
                   static_cast<cudaStream_t>(stream));
}

int b2ins_mc_free_integration_f64(const b2ins_mc_config* cfg, const double* ref_gyro,
                                  const double* ref_accel, const double* ref_nav,
                                  const double* ini, double* end_err, double* end_state,
                                  double* proc_stats, double* dump_att, double* dump_pos,
                                  double* dump_vel, double* dump_gyro, double* dump_accel,
                                  void* stream) {
  return b2ins_mc_free_integration_ex_f64(cfg, B2INS_POS_FRAME_LLA, ref_gyro, ref_accel, ref_nav, ini, end_err,
                                          end_state, proc_stats, dump_att, dump_pos, dump_vel, dump_gyro,
                                          dump_accel, stream);
}

int b2ins_mc_free_integration_f64_host(const b2ins_mc_config* cfg, const double* ref_gyro,
                                       const double* ref_accel, const double* ref_nav,
                                       const double* ini, double* end_err, double* stats) {
  ARG_CHECK(cfg, "cfg is null");
  ARG_CHECK(cfg->runs > 0 && cfg->n > 0, "runs and n must be positive");
  ARG_CHECK(ref_gyro && ref_accel && ref_nav && ini && stats, "null buffer");
  ARG_CHECK(cfg->vib_gyro.type != B2INS_VIB_SERIES && cfg->vib_accel.type != B2INS_VIB_SERIES,
            "VIB_SERIES takes a device pointer: use the device entry point");
  ARG_CHECK(cfg->ini_sets >= 1 && (cfg->ini_rows == 9 || cfg->ini_rows == 10),
            "ini must be [sets>=1][9|10]");
  const int64_t ref = cfg->n * 3;
  Staging st;
  const double* rg = st.in(ref_gyro, ref);
  const double* ra = st.in(ref_accel, ref);
  const double* rn = st.in(ref_nav, ref * 3);
  const double* di = st.in(ini, int64_t(cfg->ini_sets) * cfg->ini_rows);
  double* de = st.out(end_err, cfg->runs * 9);    // the statistics' input: on the device even if end_err is null
  double* ds = st.out(stats, 27);
  void* ws = st.scratch(b2ins_error_stats_workspace_bytes(9));
  b2ins_mc_config c = *cfg;
  c.stats_start = -1;
  c.dump_runs = 0;
  return st.run([&](cudaStream_t s) {
    const int rc = b2ins_mc_free_integration_f64(&c, rg, ra, rn, di, de, nullptr, nullptr, nullptr, nullptr,
                                                 nullptr, nullptr, nullptr, s);
    return rc != B2INS_OK ? rc : b2ins_error_stats_f64(cfg->runs, 9, de, ds, ws, s);
  });
}

// ---------------------------------------------------------------- plan ------
struct b2ins_mc_plan {
  int64_t n = 0, max_runs = 0;
  int ini_sets = 0, ini_rows = 0, device = 0;
  cudaStream_t stream = nullptr;
  double* d_in = nullptr;    // [n*3 gyro][n*3 accel][n*9 nav][sets*rows ini]
  double* d_out = nullptr;   // [27 stats][max_runs*9 end_err]
  double* d_ws = nullptr;
  double* h_in = nullptr;    // pinned: [n*3][n*3][9 last nav row][sets*rows]
  double* h_out = nullptr;   // pinned: [27][max_runs*9]
  // sub-buffers start on 16-byte boundaries (bulk async copies): offsets in doubles
  size_t n3p() const { return (static_cast<size_t>(n) * 3 + 1) & ~size_t(1); }
  size_t n9p() const { return (static_cast<size_t>(n) * 9 + 1) & ~size_t(1); }
  size_t in_doubles() const { return 2 * n3p() + n9p() + static_cast<size_t>(ini_sets) * ini_rows; }
};

int b2ins_mc_plan_destroy(b2ins_mc_plan* plan) {
  if (!plan) return B2INS_OK;
  if (plan->d_in) cudaFree(plan->d_in);
  if (plan->d_out) cudaFree(plan->d_out);
  if (plan->d_ws) cudaFree(plan->d_ws);
  if (plan->h_in) cudaFreeHost(plan->h_in);
  if (plan->h_out) cudaFreeHost(plan->h_out);
  if (plan->stream) cudaStreamDestroy(plan->stream);
  delete plan;
  return B2INS_OK;
}

int b2ins_mc_plan_create(int64_t n, int64_t max_runs, int ini_sets, int ini_rows,
                         b2ins_mc_plan** out) {
  ARG_CHECK(out, "null plan pointer");
  *out = nullptr;
  ARG_CHECK(n > 0 && max_runs > 0, "n and max_runs must be positive");
  ARG_CHECK(n < (int64_t(1) << 32), "n must be < 2^32");
  ARG_CHECK(ini_sets >= 1 && (ini_rows == 9 || ini_rows == 10), "ini must be [sets>=1][9|10]");
  b2ins_mc_plan* p = new b2ins_mc_plan();
  p->n = n;
  p->max_runs = max_runs;
  p->ini_sets = ini_sets;
  p->ini_rows = ini_rows;
  const size_t in_bytes = p->in_doubles() * sizeof(double);
  const size_t stage_bytes = (2 * p->n3p() + 10 + static_cast<size_t>(ini_sets) * ini_rows) * sizeof(double);
  const size_t out_bytes = (27 + static_cast<size_t>(max_runs) * 9) * sizeof(double);
  cudaError_t e = cudaGetDevice(&p->device);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMalloc(&p->d_in, in_bytes + 64);
  if (e == cudaSuccess) e = cudaMalloc(&p->d_out, out_bytes);
  if (e == cudaSuccess) e = cudaMalloc(&p->d_ws, static_cast<size_t>(b2ins_error_stats_workspace_bytes(9)));
  if (e == cudaSuccess) e = cudaMallocHost(&p->h_in, stage_bytes);
  if (e == cudaSuccess) e = cudaMallocHost(&p->h_out, out_bytes);
  if (e != cudaSuccess) {
    b2ins_mc_plan_destroy(p);
    return fail(B2INS_ERR_CUDA, "plan allocation failed: %s", cudaGetErrorString(e));
  }
  *out = p;
  return B2INS_OK;
}

int b2ins_mc_plan_run(b2ins_mc_plan* plan, const b2ins_mc_config* cfg, const double* ref_gyro,
                      const double* ref_accel, const double* ref_nav_end, const double* ini,
                      double* end_err, double* stats) {
  ARG_CHECK(plan && cfg, "null plan / cfg");
  ARG_CHECK(cfg->n == plan->n && cfg->runs >= 1 && cfg->runs <= plan->max_runs &&
                cfg->ini_sets == plan->ini_sets && cfg->ini_rows == plan->ini_rows,
            "cfg does not fit the plan (n=%lld runs<=%lld ini=[%d][%d])",
            static_cast<long long>(plan->n), static_cast<long long>(plan->max_runs), plan->ini_sets,
            plan->ini_rows);
  ARG_CHECK(ref_gyro && ref_accel && ref_nav_end && ini, "null buffer");
  ARG_CHECK(cfg->stats_start < 0 && cfg->dump_runs == 0,
            "a plan computes end-point errors and their statistics only");
  const int64_t n = plan->n;
  const size_t n3 = static_cast<size_t>(n) * 3;
  const size_t ini_d = static_cast<size_t>(plan->ini_sets) * plan->ini_rows;
  // stage: gyro | accel | last nav row | ini  (gyro/accel at the device offsets)
  const size_t n3p = plan->n3p();
  std::memcpy(plan->h_in, ref_gyro, n3 * sizeof(double));
  std::memcpy(plan->h_in + n3p, ref_accel, n3 * sizeof(double));
  // one slack double keeps the (virtual) base of the navigation rows 16-byte aligned
  const size_t nav_at = 2 * n3p + ((static_cast<size_t>(n - 1) * 9) & 1);
  std::memcpy(plan->h_in + nav_at, ref_nav_end, 9 * sizeof(double));
  std::memcpy(plan->h_in + nav_at + 9, ini, ini_d * sizeof(double));
  // the device block mirrors the staging block (gyro | accel | last nav row | ini): ONE copy.  The
  // kernel only reads row n-1 of the navigation rows (end-point errors), so their base pointer is
  // set n-1 rows below the staged row; the rest of the [n][9] block is never touched.
  double* d_gyro = plan->d_in;
  double* d_accel = plan->d_in + n3p;
  double* d_nav_end = plan->d_in + nav_at;
  double* d_nav = d_nav_end - (n - 1) * 9;
  double* d_ini = d_nav_end + 9;
  CU_CHECK(cudaMemcpyAsync(d_gyro, plan->h_in, (nav_at + 9 + ini_d) * sizeof(double),
                           cudaMemcpyHostToDevice, plan->stream));
  double* d_stats = plan->d_out;
  double* d_err = plan->d_out + 27;
  int rc = b2ins_mc_free_integration_f64(cfg, d_gyro, d_accel, d_nav, d_ini, d_err, nullptr,
                                         nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                                         plan->stream);
  if (rc != B2INS_OK) return rc;
  if (stats) {
    rc = b2ins_error_stats_f64(cfg->runs, 9, d_err, d_stats, plan->d_ws, plan->stream);
    if (rc != B2INS_OK) return rc;
  }
  const size_t out_d = 27 + (end_err ? static_cast<size_t>(cfg->runs) * 9 : 0);
  CU_CHECK(cudaMemcpyAsync(plan->h_out, plan->d_out, out_d * sizeof(double), cudaMemcpyDeviceToHost,
                           plan->stream));
  CU_CHECK(cudaStreamSynchronize(plan->stream));
  if (stats) std::memcpy(stats, plan->h_out, 27 * sizeof(double));
  if (end_err) std::memcpy(end_err, plan->h_out + 27, static_cast<size_t>(cfg->runs) * 9 * sizeof(double));
  return B2INS_OK;
}

double* b2ins_mc_plan_err_device(b2ins_mc_plan* plan) { return plan ? plan->d_out + 27 : nullptr; }
void* b2ins_mc_plan_stream(b2ins_mc_plan* plan) { return plan ? plan->stream : nullptr; }

// ---------------------------------------------------------------- K7 --------
static int ekf_run_bias(const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, double* rb, bool* any);
static int ekf_params(const b2ins_ekf_config* cfg, const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                      const double* rb, int ndump, EkfParams* out);
static int ekf_align_params(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, EkfParams* p);

int b2ins_ins_loose_f64(const b2ins_ekf_config* cfg, const double* ref_gyro, const double* ref_accel,
                        const double* ref_nav, const double* ref_gps, const int64_t* gps_idx,
                        const double* gps_vis, double* end_err, double* end_bias, double* consist,
                        double* dump_att, double* dump_pos, double* dump_vel, double* dump_wb,
                        double* dump_ab, void* stream) {
  return b2ins_ins_loose_ex_f64(cfg, nullptr, nullptr, ref_gyro, ref_accel, ref_nav, ref_gps, gps_idx, gps_vis,
                                end_err, end_bias, consist, dump_att, dump_pos, dump_vel, dump_wb, dump_ab, stream);
}

int b2ins_ins_loose_ex_f64(const b2ins_ekf_config* cfg, const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                           const double* ref_gyro, const double* ref_accel, const double* ref_nav,
                           const double* ref_gps, const int64_t* gps_idx, const double* gps_vis, double* end_err,
                           double* end_bias, double* consist, double* dump_att, double* dump_pos,
                           double* dump_vel, double* dump_wb, double* dump_ab, void* stream) {
  return b2ins_ins_loose_rx_f64(cfg, nullptr, vib_gyro, vib_accel, -1, B2INS_POS_FRAME_LLA, ref_gyro, ref_accel,
                                ref_nav, ref_gps, gps_idx, gps_vis, end_err, end_bias, consist, nullptr, dump_att,
                                dump_pos, dump_vel, dump_wb, dump_ab, nullptr, nullptr, nullptr, stream);
}

int b2ins_ins_loose_proc_f64(const b2ins_ekf_config* cfg, const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                             int64_t proc_start, int proc_pos_frame, const double* ref_gyro, const double* ref_accel,
                             const double* ref_nav, const double* ref_gps, const int64_t* gps_idx,
                             const double* gps_vis, double* end_err, double* end_bias, double* consist,
                             double* proc_stats, double* dump_att, double* dump_pos, double* dump_vel,
                             double* dump_wb, double* dump_ab, void* stream) {
  ARG_CHECK(cfg, "cfg is null");
  ARG_CHECK(proc_pos_frame >= B2INS_POS_FRAME_LLA && proc_pos_frame <= B2INS_POS_FRAME_ECEF,
            "proc_pos_frame must be B2INS_POS_FRAME_*");
  ARG_CHECK(proc_stats, "null buffer: proc_stats is required");
  ARG_CHECK(proc_start >= 0 && proc_start < cfg->n, "proc_start must be in [0, n)");
  return b2ins_ins_loose_rx_f64(cfg, nullptr, vib_gyro, vib_accel, proc_start, proc_pos_frame, ref_gyro, ref_accel,
                                ref_nav, ref_gps, gps_idx, gps_vis, end_err, end_bias, consist, proc_stats, dump_att,
                                dump_pos, dump_vel, dump_wb, dump_ab, nullptr, nullptr, nullptr, stream);
}

int b2ins_ins_loose_align_f64(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, const b2ins_vib* vib_gyro,
                              const b2ins_vib* vib_accel, int64_t proc_start, int proc_pos_frame,
                              const double* ref_gyro, const double* ref_accel, const double* ref_nav,
                              const double* ref_gps, const int64_t* gps_idx, const double* gps_vis, double* end_err,
                              double* end_bias, double* consist, double* proc_stats, double* dump_att,
                              double* dump_pos, double* dump_vel, double* dump_wb, double* dump_ab, void* stream) {
  return b2ins_ins_loose_rx_f64(cfg, align, vib_gyro, vib_accel, proc_start, proc_pos_frame, ref_gyro, ref_accel,
                                ref_nav, ref_gps, gps_idx, gps_vis, end_err, end_bias, consist, proc_stats, dump_att,
                                dump_pos, dump_vel, dump_wb, dump_ab, nullptr, nullptr, nullptr, stream);
}

// K7 on generated measurements, the launch site of every generated form: ekf_kernel<VIB, false, PROC> (PROC:
// proc_stats given), and with a turn-on bias or end_bias_err its RB form
int b2ins_ins_loose_rx_f64(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, const b2ins_vib* vib_gyro,
                           const b2ins_vib* vib_accel, int64_t proc_start, int proc_pos_frame,
                           const double* ref_gyro, const double* ref_accel, const double* ref_nav,
                           const double* ref_gps, const int64_t* gps_idx, const double* gps_vis, double* end_err,
                           double* end_bias, double* consist, double* proc_stats, double* dump_att,
                           double* dump_pos, double* dump_vel, double* dump_wb, double* dump_ab,
                           const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, double* end_bias_err,
                           void* stream) {
  ARG_CHECK(cfg, "cfg is null");
  if (proc_stats) {
    ARG_CHECK(proc_pos_frame >= B2INS_POS_FRAME_LLA && proc_pos_frame <= B2INS_POS_FRAME_ECEF,
              "proc_pos_frame must be B2INS_POS_FRAME_*");
    ARG_CHECK(proc_start >= 0 && proc_start < cfg->n, "proc_start must be in [0, n)");
  }
  ARG_CHECK((proc_stats == nullptr) == (proc_start == -1), "proc_stats and proc_start >= 0 must be given together");
  double rb[6];
  bool any_rb;
  int rc = ekf_run_bias(gyro_run, accel_run, rb, &any_rb);
  if (rc != B2INS_OK) return rc;
  ARG_CHECK(cfg->fs > 0.0, "fs must be positive");
  ARG_CHECK(cfg->runs >= 0 && cfg->n >= 0 && cfg->m >= 0, "runs, n and m must be non-negative");
  if (cfg->runs == 0 || cfg->n == 0) return B2INS_OK;
  ARG_CHECK(cfg->n < (int64_t(1) << 32), "n must be < 2^32");
  ARG_CHECK(ref_gyro && ref_accel && ref_nav && end_err, "null buffer");
  ARG_CHECK(cfg->m == 0 || (ref_gps && gps_idx && gps_vis), "m > 0 needs ref_gps, gps_idx and gps_vis");
  ARG_CHECK(cfg->dump_runs >= 0 && cfg->dump_runs <= cfg->runs, "dump_runs out of range");
  const int ndump = (dump_att != nullptr) + (dump_pos != nullptr) + (dump_vel != nullptr) + (dump_wb != nullptr) +
                    (dump_ab != nullptr);
  ARG_CHECK(ndump == 0 || ndump == 5, "dump_att/pos/vel/wb/ab must be given together");
  ARG_CHECK(cfg->dump_stride >= 0, "dump_stride must be >= 0");
  EkfParams p;
  rc = ekf_params(cfg, vib_gyro, vib_accel, rb, ndump, &p);
  if (rc != B2INS_OK) return rc;
  rc = ekf_align_params(cfg, align, &p);
  if (rc != B2INS_OK) return rc;
  p.ref_gyro = ref_gyro;
  p.ref_accel = ref_accel;
  p.ref_nav = ref_nav;
  p.ref_gps = ref_gps;
  p.gps_idx = gps_idx;
  p.gps_vis = gps_vis;
  p.stats_start = cfg->stats_start;
  p.end_err = end_err;
  p.end_bias = end_bias;
  p.consist = consist;
  p.out_att = dump_att;
  p.out_pos = dump_pos;
  p.out_vel = dump_vel;
  p.out_wb = dump_wb;
  p.out_ab = dump_ab;
  p.proc_stats = proc_stats;
  p.proc_start = proc_start;
  p.proc_pos_frame = proc_pos_frame;
  p.end_bias_err = end_bias_err;
  const unsigned grid = static_cast<unsigned>((cfg->runs + kEkfRuns - 1) / kEkfRuns);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool vib = !(p.gyro.vib_type == B2INS_VIB_NONE && p.accel.vib_type == B2INS_VIB_NONE);
  if (any_rb || end_bias_err) {
    if (proc_stats) {
      if (vib)
        ekf_kernel<true, false, true, false, true><<<grid, kEkfThreads, 0, s>>>(p);
      else
        ekf_kernel<false, false, true, false, true><<<grid, kEkfThreads, 0, s>>>(p);
    } else {
      if (vib)
        ekf_kernel<true, false, false, false, true><<<grid, kEkfThreads, 0, s>>>(p);
      else
        ekf_kernel<false, false, false, false, true><<<grid, kEkfThreads, 0, s>>>(p);
    }
  } else if (proc_stats) {
    if (vib)
      ekf_kernel<true, false, true><<<grid, kEkfThreads, 0, s>>>(p);
    else
      ekf_kernel<false, false, true><<<grid, kEkfThreads, 0, s>>>(p);
  } else {
    if (vib)
      ekf_kernel<true, false, false><<<grid, kEkfThreads, 0, s>>>(p);
    else
      ekf_kernel<false, false, false><<<grid, kEkfThreads, 0, s>>>(p);
  }
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_ins_loose_fed_f64(const b2ins_ekf_config* cfg, int ini_draw, const double* gyro, const double* accel,
                            const double* gps, const int64_t* gps_idx, const double* gps_vis,
                            const double* ref_nav, double* end_err, double* end_bias, double* dump_att,
                            double* dump_pos, double* dump_vel, double* dump_wb, double* dump_ab, void* stream) {
  return b2ins_ins_loose_fed_rx_f64(cfg, nullptr, ini_draw, gyro, accel, gps, gps_idx, gps_vis, ref_nav, end_err,
                                    end_bias, dump_att, dump_pos, dump_vel, dump_wb, dump_ab, nullptr, nullptr, stream);
}

int b2ins_ins_loose_fed_align_f64(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, const double* gyro,
                                  const double* accel, const double* gps, const int64_t* gps_idx,
                                  const double* gps_vis, const double* ref_nav, double* end_err, double* end_bias,
                                  double* dump_att, double* dump_pos, double* dump_vel, double* dump_wb,
                                  double* dump_ab, void* stream) {
  return b2ins_ins_loose_fed_rx_f64(cfg, align, 0, gyro, accel, gps, gps_idx, gps_vis, ref_nav, end_err, end_bias,
                                    dump_att, dump_pos, dump_vel, dump_wb, dump_ab, nullptr, nullptr, stream);
}

// K7 on supplied measurements, the launch site of every fed form (ekf_kernel<false, true, false, aligned>); the
// turn-on bias is in the data and enters the model through P0 only
int b2ins_ins_loose_fed_rx_f64(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, int ini_draw,
                               const double* gyro, const double* accel, const double* gps, const int64_t* gps_idx,
                               const double* gps_vis, const double* ref_nav, double* end_err, double* end_bias,
                               double* dump_att, double* dump_pos, double* dump_vel, double* dump_wb, double* dump_ab,
                               const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, void* stream) {
  ARG_CHECK(cfg, "cfg is null");
  ARG_CHECK(cfg->fs > 0.0, "fs must be positive");
  ARG_CHECK(cfg->runs >= 0 && cfg->n >= 0 && cfg->m >= 0, "runs, n and m must be non-negative");
  ARG_CHECK(ini_draw == 0 || ini_draw == 1, "ini_draw must be 0 or 1");
  ARG_CHECK(ini_draw == 0 || !align || align->mode == B2INS_ALIGN_OFF, "an aligned filter makes no initial draw");
  ARG_CHECK((end_err == nullptr) == (ref_nav == nullptr), "end_err and ref_nav must be given together");
  double rb[6];
  bool any_rb;
  int rc = ekf_run_bias(gyro_run, accel_run, rb, &any_rb);
  if (rc != B2INS_OK) return rc;
  if (cfg->runs == 0 || cfg->n == 0) return B2INS_OK;
  ARG_CHECK(cfg->n < (int64_t(1) << 32), "n must be < 2^32");
  ARG_CHECK(gyro && accel, "null buffer: gyro and accel are required");
  ARG_CHECK(cfg->m == 0 || (gps && gps_idx && gps_vis), "m > 0 needs gps, gps_idx and gps_vis");
  ARG_CHECK(cfg->dump_runs >= 0 && cfg->dump_runs <= cfg->runs, "dump_runs out of range");
  const int ndump = (dump_att != nullptr) + (dump_pos != nullptr) + (dump_vel != nullptr) + (dump_wb != nullptr) +
                    (dump_ab != nullptr);
  ARG_CHECK(ndump == 0 || ndump == 5, "dump_att/pos/vel/wb/ab must be given together");
  ARG_CHECK(cfg->dump_stride >= 0, "dump_stride must be >= 0");
  EkfParams p;
  rc = ekf_params(cfg, nullptr, nullptr, rb, ndump, &p);
  if (rc != B2INS_OK) return rc;
  rc = ekf_align_params(cfg, align, &p);
  if (rc != B2INS_OK) return rc;
  p.ref_nav = ref_nav;
  p.gps_idx = gps_idx;
  p.gps_vis = gps_vis;
  p.fed_gyro = gyro;
  p.fed_accel = accel;
  p.fed_gps = gps;
  p.ini_draw = ini_draw;
  p.end_err = end_err;
  p.end_bias = end_bias;
  p.out_att = dump_att;
  p.out_pos = dump_pos;
  p.out_vel = dump_vel;
  p.out_wb = dump_wb;
  p.out_ab = dump_ab;
  const unsigned grid = static_cast<unsigned>((cfg->runs + kEkfRuns - 1) / kEkfRuns);
  if (p.align)
    ekf_kernel<false, true, false, true><<<grid, kEkfThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  else
    ekf_kernel<false, true, false, false><<<grid, kEkfThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

// The turn-on bias of the run errors for K7: rb = the 1-sigma per generator channel (accel x y z, gyro x y z), zero
// for a null struct; *any is false when all are zero.  The filter's states hold a bias but no scale factor or
// misalignment, so sf and ma must be zero; b is checked as digest_run_err checks it.
static int ekf_run_bias(const b2ins_run_err* gyro_run, const b2ins_run_err* accel_run, double* rb, bool* any) {
  RunErrs re;
  bool unused;
  const int rc = digest_run_err(gyro_run, accel_run, &re, &unused);
  if (rc != B2INS_OK) return rc;
  *any = false;
  for (int s = 0; s < 2; ++s) {
    for (int c = 0; c < 3; ++c) {
      ARG_CHECK(re.s[s].sf[c] == 0.0, "the loosely-coupled filter takes no run-to-run scale factor: sf must be 0");
      for (int j = 0; j < 3; ++j)
        ARG_CHECK(re.s[s].ma[c][j] == 0.0, "the loosely-coupled filter takes no run-to-run misalignment: ma must be 0");
      rb[3 * s + c] = re.s[s].b[c];
      *any = *any || rb[3 * s + c] != 0.0;
    }
  }
  return B2INS_OK;
}

// The filter model of cfg (Q, R, P0, bias model, initial state) and the launch geometry of K7; the
// caller sets the buffers.  vib_*: the generator's vibration (NULL for supplied measurements); rb: the turn-on
// bias sigmas of ekf_run_bias.
static int ekf_params(const b2ins_ekf_config* cfg, const b2ins_vib* vib_gyro, const b2ins_vib* vib_accel,
                      const double* rb, int ndump, EkfParams* out) {
  EkfParams& p = *out;
  std::memset(&p, 0, sizeof(p));
  p.n = cfg->n;
  p.runs = cfg->runs;
  p.run_offset = cfg->run_offset;
  p.m = cfg->m;
  p.dt = 1.0 / cfg->fs;
  p.earth_rot = cfg->earth_rot;
  p.k0 = static_cast<uint32_t>(cfg->seed);
  p.k1 = static_cast<uint32_t>(cfg->seed >> 32);
  int rc = digest_triad(&cfg->gyro_err, vib_gyro, cfg->fs, &p.gyro);
  if (rc != B2INS_OK) return rc;
  rc = digest_triad(&cfg->accel_err, vib_accel, cfg->fs, &p.accel);
  if (rc != B2INS_OK) return rc;
  for (int c = 0; c < 3; ++c) {
    p.stdp[c] = cfg->gps_stdp[c];
    p.stdv[c] = cfg->gps_stdv[c];
    p.p0[c] = cfg->gps_stdp[c] * cfg->gps_stdp[c];
    p.p0[3 + c] = cfg->gps_stdv[c] * cfg->gps_stdv[c];
    p.p0[6 + c] = cfg->ini_att_std[c] * cfg->ini_att_std[c];
    // the bias states: the drift, the constant bias the filter does not know and the run's turn-on bias
    p.rb[c] = rb[c];
    p.rb[3 + c] = rb[3 + c];
    p.p0[9 + c] = cfg->gyro_err.b_drift[c] * cfg->gyro_err.b_drift[c] + cfg->gyro_err.b[c] * cfg->gyro_err.b[c] +
                  rb[3 + c] * rb[3 + c];
    p.p0[12 + c] = cfg->accel_err.b_drift[c] * cfg->accel_err.b_drift[c] + cfg->accel_err.b[c] * cfg->accel_err.b[c] +
                   rb[c] * rb[c];
    // the filter's bias model is the generator's: a = 1 - dt/tau, b^2 (white drift: a = 0, b = drift)
    const bool wg = std::isinf(cfg->gyro_err.b_corr[c]), wa = std::isinf(cfg->accel_err.b_corr[c]);
    p.ag[c] = wg ? 0.0 : p.gyro.gm_a[c];
    p.qg[c] = wg ? p.gyro.wd[c] * p.gyro.wd[c] : p.gyro.gm_b[c] * p.gyro.gm_b[c];
    p.aa[c] = wa ? 0.0 : p.accel.gm_a[c];
    p.qa[c] = wa ? p.accel.wd[c] * p.accel.wd[c] : p.accel.gm_b[c] * p.accel.gm_b[c];
    p.arw2dt[c] = cfg->gyro_err.rw[c] * cfg->gyro_err.rw[c] * p.dt;
    p.vrw2dt[c] = cfg->accel_err.rw[c] * cfg->accel_err.rw[c] * p.dt;
  }
  for (int c = 0; c < 9; ++c) p.ini[c] = cfg->ini[c];
  ARG_CHECK(cfg->vel_rw >= 0.0 && cfg->att_rw >= 0.0, "vel_rw and att_rw must be >= 0");
  p.qv_extra = cfg->vel_rw * cfg->vel_rw * p.dt;
  p.qphi_extra = cfg->att_rw * cfg->att_rw * p.dt;
  p.dump_runs = ndump ? cfg->dump_runs : 0;
  p.dump_stride = cfg->dump_stride > 1 ? cfg->dump_stride : 1;
  p.dump_rows = (cfg->n + p.dump_stride - 1) / p.dump_stride;
  return B2INS_OK;
}

// The alignment of b2ins_ekf_align (NULL: off) into p: the mode, the given yaw and the P0 terms that are the
// same for every run (include/b2ins.h).  Accelerometer y sets roll (the N misalignment), x sets pitch (E).
static int ekf_align_params(const b2ins_ekf_config* cfg, const b2ins_ekf_align* align, EkfParams* p) {
  p->align = align ? align->mode : B2INS_ALIGN_OFF;
  if (p->align == B2INS_ALIGN_OFF) return B2INS_OK;
  ARG_CHECK(p->align == B2INS_ALIGN_YAW || p->align == B2INS_ALIGN_GPS, "align->mode must be B2INS_ALIGN_*");
  static_assert(kAlignGps == B2INS_ALIGN_GPS, "the kernel's GPS-heading mode");
  ARG_CHECK(cfg->n == 0 || cfg->n >= kAlignN, "alignment needs n >= 10 IMU samples");
  ARG_CHECK(std::isfinite(align->yaw) || p->align == B2INS_ALIGN_GPS, "align->yaw must be finite");
  ARG_CHECK(align->yaw_var >= 0.0 || p->align == B2INS_ALIGN_GPS, "align->yaw_var must be >= 0");
  constexpr double kG = 9.80665;
  const b2ins_sensor_err& a = cfg->accel_err;
  for (int c = 0; c < 2; ++c) {
    const int ax = 1 - c;
    p->align_p0[c] = (a.b[ax] * a.b[ax] + a.b_drift[ax] * a.b_drift[ax] + p->rb[ax] * p->rb[ax] +
                      a.rw[ax] * a.rw[ax] * cfg->fs / kAlignN) /
                     (kG * kG);
  }
  p->align_yaw = align->yaw;
  p->align_p0[2] = align->yaw_var;
  for (int c = 0; c < 3; ++c) p->arw2[c] = cfg->gyro_err.rw[c] * cfg->gyro_err.rw[c];
  return B2INS_OK;
}

// ---------------------------------------------------------------- K3 --------
int64_t b2ins_error_stats_workspace_bytes(int ncomp) {
  if (ncomp < 1) return 0;
  // per-block partials + partial[2nc] + mean... : [kStatBlocks][2][nc] + 4*nc
  return static_cast<int64_t>(sizeof(double)) * (static_cast<int64_t>(kStatBlocks) * 2 + 4) * ncomp;
}

static int stage1_grid(int64_t runs, int ncomp, int threads) {
  const int64_t total = runs * ncomp;
  int64_t g = (total + threads - 1) / threads;
  if (g > kStatBlocks) g = kStatBlocks;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}

int b2ins_error_partial_f64(int64_t runs, int ncomp, const double* err, double* partial,
                            void* workspace, void* stream) {
  ARG_CHECK(runs > 0 && ncomp >= 1 && ncomp <= kStatMaxComp, "bad runs/ncomp");
  ARG_CHECK(err && partial && workspace, "null buffer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int threads = stat_threads(ncomp);
  const int grid = stage1_grid(runs, ncomp, threads);
  double* ws = static_cast<double*>(workspace);
  err_stage1_kernel<0><<<grid, threads, 2 * threads * sizeof(double), s>>>(runs, ncomp, err,
                                                                           nullptr, ws);
  err_stage2_kernel<0><<<1, 32, 0, s>>>(grid, ncomp, ws, partial);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_error_partial2_f64(int64_t runs, int ncomp, const double* err, const double* mean,
                             double* partial2, void* workspace, void* stream) {
  ARG_CHECK(runs > 0 && ncomp >= 1 && ncomp <= kStatMaxComp, "bad runs/ncomp");
  ARG_CHECK(err && mean && partial2 && workspace, "null buffer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int threads = stat_threads(ncomp);
  const int grid = stage1_grid(runs, ncomp, threads);
  double* ws = static_cast<double*>(workspace);
  err_stage1_kernel<1><<<grid, threads, 2 * threads * sizeof(double), s>>>(runs, ncomp, err, mean,
                                                                           ws);
  err_stage2_kernel<1><<<1, 32, 0, s>>>(grid, ncomp, ws, partial2);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_error_stats_f64(int64_t runs, int ncomp, const double* err, double* stats,
                          void* workspace, void* stream) {
  ARG_CHECK(runs > 0 && ncomp >= 1 && ncomp <= kStatMaxComp, "bad runs/ncomp");
  ARG_CHECK(err && stats && workspace, "null buffer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (runs * ncomp <= kStatSmallMax) {
    stats_small_kernel<<<1, kStatSmallThreads, 0, s>>>(runs, ncomp, err, stats);
    CU_CHECK(cudaGetLastError());
    return B2INS_OK;
  }
  double* ws = static_cast<double*>(workspace);
  double* partial = ws + static_cast<int64_t>(kStatBlocks) * 2 * ncomp;  // [2nc]
  double* partial2 = partial + 2 * ncomp;                                // [nc]
  int rc = b2ins_error_partial_f64(runs, ncomp, err, partial, workspace, stream);
  if (rc != B2INS_OK) return rc;
  stats_mean_kernel<<<1, 32, 0, s>>>(runs, ncomp, partial, stats);
  rc = b2ins_error_partial2_f64(runs, ncomp, err, stats + ncomp, partial2, workspace, stream);
  if (rc != B2INS_OK) return rc;
  stats_std_kernel<<<1, 32, 0, s>>>(runs, ncomp, partial2, stats);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_error_stats_exchange_f64(int64_t runs, int ncomp, const double* err, int rank, int world,
                                   const uint64_t* windows, uint64_t seq, double* stats,
                                   int* timeout_flag, void* stream) {
  ARG_CHECK(runs >= 0 && ncomp >= 1 && 3 * ncomp + 2 <= kXchgSlot, "bad runs/ncomp");
  ARG_CHECK(runs * ncomp <= kStatSmallMax, "the fused exchange handles runs*ncomp <= 2^17 per rank");
  ARG_CHECK(world >= 1 && world <= kXchgMaxWorld && rank >= 0 && rank < world, "bad rank/world");
  ARG_CHECK(windows && stats && timeout_flag && seq >= 1, "null buffer / seq must start at 1");
  ARG_CHECK(runs == 0 || err, "null err");
  XchgParams p;
  std::memset(&p, 0, sizeof(p));
  p.runs = runs;
  p.ncomp = ncomp;
  p.rank = rank;
  p.world = world;
  p.seq = seq;
  p.err = err;
  for (int q = 0; q < world; ++q) p.peer[q] = reinterpret_cast<double*>(windows[q]);
  p.out = stats;
  p.timeout_flag = timeout_flag;
  stats_exchange_kernel<<<1, kStatSmallThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

// ---------------------------------------------------------------- K4 --------
int64_t b2ins_allan_workspace_bytes(int64_t n, int64_t nseries) {
  return allan_workspace_bytes(n, nseries);
}

int b2ins_allan_f64(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner,
                    int64_t outer_stride, int64_t sample_stride, double* avar, double* tau,
                    void* workspace, void* stream) {
  const int chk = series_check(fs, n, nseries, inner, outer_stride, sample_stride);
  if (chk != B2INS_OK) return chk;
  int64_t mult[128];
  const int ntau = b2ins_allan_num_tau(n, fs, mult, 128);
  if (ntau == 0 || nseries == 0) return B2INS_OK;
  ARG_CHECK(ntau <= 128, "too many tau");
  ARG_CHECK(x && avar && tau && workspace, "null buffer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int rc = allan_launch(fs, n, nseries, x, inner, outer_stride, sample_stride, mult, ntau,
                              avar, tau, workspace, sm_count(), s);
  if (rc != 0) return fail(B2INS_ERR_CUDA, "allan launch failed: %s", cudaGetErrorString(cudaGetLastError()));
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_allan_mc_f64(double fs, int64_t n, int64_t runs, const double* ref_gyro,
                       const double* ref_accel, const b2ins_sensor_err* gyro_err,
                       const b2ins_sensor_err* accel_err, uint64_t seed, int64_t run_offset,
                       double* avar, double* tau, void* workspace, void* stream) {
  ARG_CHECK(fs > 0.0 && n >= 0 && runs >= 0, "bad fs/n/runs");
  int64_t mult[128];
  const int ntau = b2ins_allan_num_tau(n, fs, mult, 128);
  if (ntau == 0 || runs == 0) return B2INS_OK;
  ARG_CHECK(ntau <= 128, "too many tau");
  ARG_CHECK(n > kAllanChunk, "the fused Allan path needs more than %d samples per series", kAllanChunk);
  ARG_CHECK(n < (int64_t(1) << 32), "n must be < 2^32");
  ARG_CHECK(ref_gyro && ref_accel && gyro_err && accel_err && avar && tau && workspace, "null buffer");
  AllanGenParams g;
  std::memset(&g, 0, sizeof(g));
  g.n = n;
  g.run_offset = run_offset;
  g.k0 = static_cast<uint32_t>(seed);
  g.k1 = static_cast<uint32_t>(seed >> 32);
  int rc = digest_triad(gyro_err, nullptr, fs, &g.gyro);
  if (rc != B2INS_OK) return rc;
  rc = digest_triad(accel_err, nullptr, fs, &g.accel);
  if (rc != B2INS_OK) return rc;
  g.ref_gyro = ref_gyro;
  g.ref_accel = ref_accel;
  rc = allan_launch(fs, n, runs * 6, nullptr, 1, n, 1, mult, ntau, avar, tau, workspace, sm_count(),
                    static_cast<cudaStream_t>(stream), &g);
  if (rc != 0) return fail(B2INS_ERR_CUDA, "allan launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

// K4 and K4o's two forms from host memory: the device entry's checks, then only the span of x the series read
typedef int (*VarianceEntry)(double, int64_t, int64_t, const double*, int64_t, int64_t, int64_t, double*, double*,
                             void*, void*);

static int variance_host(VarianceEntry entry, int64_t (*workspace_bytes)(int64_t, int64_t), double fs, int64_t n,
                         int64_t nseries, const double* x, int64_t inner, int64_t outer_stride, int64_t sample_stride,
                         double* var, double* tau) {
  const int chk = series_check(fs, n, nseries, inner, outer_stride, sample_stride);
  if (chk != B2INS_OK) return chk;
  const int ntau = b2ins_allan_num_tau(n, fs, nullptr, 0);
  if (ntau == 0 || nseries == 0) return B2INS_OK;
  ARG_CHECK(x && var && tau, "null buffer");
  Staging st;
  const double* dx = st.in(x, series_elems(n, nseries, inner, outer_stride, sample_stride));
  double* dvar = st.out(var, nseries * ntau);
  double* dtau = st.out(tau, ntau);
  void* ws = st.scratch(workspace_bytes(n, nseries));
  return st.run([&](cudaStream_t s) {
    return entry(fs, n, nseries, dx, inner, outer_stride, sample_stride, dvar, dtau, ws, s);
  });
}

int b2ins_allan_f64_host(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner,
                         int64_t outer_stride, int64_t sample_stride, double* avar, double* tau) {
  return variance_host(b2ins_allan_f64, b2ins_allan_workspace_bytes, fs, n, nseries, x, inner, outer_stride,
                       sample_stride, avar, tau);
}

// ---------------------------------------------------------------- K4o -------
int64_t b2ins_oallan_workspace_bytes(int64_t n, int64_t nseries) {
  return oallan_workspace_bytes(n, nseries);
}

// K4o and its Hadamard form: one argument check and one launch; the workspace serves both
static int oallan_f64(bool hadamard, double fs, int64_t n, int64_t nseries, const double* x, int64_t inner,
                      int64_t outer_stride, int64_t sample_stride, double* avar, double* tau,
                      void* workspace, void* stream) {
  const int chk = series_check(fs, n, nseries, inner, outer_stride, sample_stride);
  if (chk != B2INS_OK) return chk;
  int64_t mult[128];
  const int ntau = b2ins_allan_num_tau(n, fs, mult, 128);
  if (ntau == 0 || nseries == 0) return B2INS_OK;
  ARG_CHECK(ntau <= 128, "too many tau");
  ARG_CHECK(x && avar && tau && workspace, "null buffer");
  const int rc = oallan_launch(fs, n, nseries, x, inner, outer_stride, sample_stride, mult, ntau, avar, tau,
                               workspace, static_cast<cudaStream_t>(stream), hadamard);
  if (rc == 4)
    return fail(B2INS_ERR_ARG, "overlapping %s: too many series x samples for one call",
                hadamard ? "Hadamard" : "Allan");
  if (rc != 0)
    return fail(B2INS_ERR_CUDA, "%s launch failed (%d): %s", hadamard ? "ohadamard" : "oallan", rc,
                cudaGetErrorString(cudaGetLastError()));
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_oallan_f64(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner,
                     int64_t outer_stride, int64_t sample_stride, double* avar, double* tau,
                     void* workspace, void* stream) {
  return oallan_f64(false, fs, n, nseries, x, inner, outer_stride, sample_stride, avar, tau, workspace, stream);
}

int b2ins_oallan_f64_host(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner,
                          int64_t outer_stride, int64_t sample_stride, double* avar, double* tau) {
  return variance_host(b2ins_oallan_f64, b2ins_oallan_workspace_bytes, fs, n, nseries, x, inner, outer_stride,
                       sample_stride, avar, tau);
}

int b2ins_ohadamard_f64(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner,
                        int64_t outer_stride, int64_t sample_stride, double* hvar, double* tau,
                        void* workspace, void* stream) {
  return oallan_f64(true, fs, n, nseries, x, inner, outer_stride, sample_stride, hvar, tau, workspace, stream);
}

int b2ins_ohadamard_f64_host(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner,
                             int64_t outer_stride, int64_t sample_stride, double* hvar, double* tau) {
  return variance_host(b2ins_ohadamard_f64, b2ins_oallan_workspace_bytes, fs, n, nseries, x, inner, outer_stride,
                       sample_stride, hvar, tau);
}

// ---------------------------------------------------------------- K13 -------
// K13's checks, shared by the device entry and its host wrapper; nseries = 0 is left to the caller.  The grid
// and the weights go to *p, from (n, fs) by K4's own grid function.
static int allan_fit_check(double fs, int64_t n, int64_t nseries, int64_t series_stride, int64_t bin_stride,
                           AllanFitParams* p) {
  ARG_CHECK(fs > 0.0 && std::isfinite(fs) && n >= 0 && nseries >= 0, "bad fs/n/nseries");
  ARG_CHECK(series_stride >= 0 && bin_stride >= 1, "bad strides");
  ARG_CHECK(nseries / kFitWarps + (nseries % kFitWarps != 0) <= INT32_MAX, "too many series for one call");
  int64_t mult[kFitMaxBins];
  const int ntau = b2ins_allan_num_tau(n, fs, mult, kFitMaxBins);
  ARG_CHECK(ntau <= kFitMaxBins, "too many tau");
  p->ntau = ntau;
  for (int k = 0; k < ntau; ++k) {
    p->tau[k] = static_cast<double>(mult[k]) * (1.0 / fs);
    p->w[k] = static_cast<double>(n / mult[k] - 1);
  }
  return B2INS_OK;
}

int b2ins_allan_fit_f64(double fs, int64_t n, int64_t nseries, const double* var, int64_t series_stride,
                        int64_t bin_stride, double* out, void* stream) {
  AllanFitParams p;
  std::memset(&p, 0, sizeof(p));
  const int chk = allan_fit_check(fs, n, nseries, series_stride, bin_stride, &p);
  if (chk != B2INS_OK) return chk;
  if (nseries == 0) return B2INS_OK;
  ARG_CHECK(out && (var || p.ntau == 0), "null buffer");
  p.var = var;
  p.out = out;
  p.nseries = nseries;
  p.series_stride = series_stride;
  p.bin_stride = bin_stride;
  p.b_scale = std::sqrt(kPi / (2.0 * std::log(2.0)));
  p.nan = std::numeric_limits<double>::quiet_NaN();
  const int64_t ctas = (nseries + kFitWarps - 1) / kFitWarps;
  allan_fit_kernel<<<static_cast<unsigned>(ctas), kFitWarps * 32, 0, static_cast<cudaStream_t>(stream)>>>(p);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

int b2ins_allan_fit_f64_host(double fs, int64_t n, int64_t nseries, const double* var, int64_t series_stride,
                             int64_t bin_stride, double* out) {
  AllanFitParams p;
  const int chk = allan_fit_check(fs, n, nseries, series_stride, bin_stride, &p);
  if (chk != B2INS_OK) return chk;
  if (nseries == 0) return B2INS_OK;
  ARG_CHECK(out && (var || p.ntau == 0), "null buffer");
  Staging st;
  const double* dv =
      p.ntau == 0 ? nullptr : st.in(var, (nseries - 1) * series_stride + (p.ntau - 1) * bin_stride + 1);
  double* dout = st.out(out, nseries * 6);
  return st.run([&](cudaStream_t s) {
    return b2ins_allan_fit_f64(fs, n, nseries, dv, series_stride, bin_stride, dout, s);
  });
}

// ---------------------------------------------------------------- K5 --------
// B2INS_PSD_DIRECT (tools: A/B the two paths) forces the direct synthesis; read once per process, so a
// launch and b2ins_diag_psd_plan always agree
static bool psd_direct_forced() {
  static const bool forced = std::getenv("B2INS_PSD_DIRECT") != nullptr;
  return forced;
}

int b2ins_psd_series_len(int64_t n) { return n > 0 ? psd_series_len(n) : 0; }

int b2ins_diag_psd_plan(int64_t n, int* P) {
  if (n <= 0 || !P) {
    fail(B2INS_ERR_ARG, "bad n or null output");
    return -1;
  }
  int bluestein = 0;
  const int len = psd_direct_forced() ? 0 : psd_fft_plan(psd_series_len(n), &bluestein);
  *P = len;
  return len == 0 ? 0 : (bluestein ? 2 : 1);
}

// ---------------------------------------------------------------- K11 -------
// [0, 16): the bin scale; then K5's chirp transform (Bluestein, P <= 8192 complex); then the chunk sums
static int64_t welch_partial_offset(const WelchPlan& w) { return 16 + (w.bluestein ? int64_t(w.P) * 16 : 0); }

int64_t b2ins_welch_workspace_bytes(int64_t n, int64_t nseries, int64_t nperseg, int64_t noverlap) {
  WelchPlan w;
  if (nseries < 0 || !welch_plan(n, nperseg, noverlap, &w)) return -1;
  const int64_t parts = w.nchunk > 1 ? nseries * w.nchunk * (w.M + 1) * 8 : 0;
  return welch_partial_offset(w) + parts;
}

// K11's checks, shared by the device entry and its host wrapper.  K11 words its own rate and length rules, so
// the common series check comes after them and only its stride rule can still fail there.
static int welch_check(double fs, int64_t n, int64_t nseries, int64_t inner, int64_t outer_stride,
                       int64_t sample_stride, int64_t nperseg, int64_t noverlap, WelchPlan* w) {
  ARG_CHECK(fs > 0.0 && std::isfinite(fs) && nseries >= 0, "bad fs/nseries");
  ARG_CHECK(noverlap >= 0 && noverlap < nperseg, "need 0 <= noverlap < nperseg, got noverlap=%lld, nperseg=%lld",
            static_cast<long long>(noverlap), static_cast<long long>(nperseg));
  ARG_CHECK(n >= nperseg, "a series of %lld samples is shorter than nperseg=%lld", static_cast<long long>(n),
            static_cast<long long>(nperseg));
  const int chk = series_check(fs, n, nseries, inner, outer_stride, sample_stride);
  if (chk != B2INS_OK) return chk;
  ARG_CHECK(welch_plan(n, nperseg, noverlap, w),
            "nperseg=%lld: need an even length >= 16, a power of two up to 16384 or at most 8192",
            static_cast<long long>(nperseg));
  return B2INS_OK;
}

int b2ins_welch_f64(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner, int64_t outer_stride,
                    int64_t sample_stride, int64_t nperseg, int64_t noverlap, const double* window, double* psd,
                    double* freq, void* workspace, void* stream) {
  WelchPlan w;
  const int chk = welch_check(fs, n, nseries, inner, outer_stride, sample_stride, nperseg, noverlap, &w);
  if (chk != B2INS_OK) return chk;
  ARG_CHECK(window && freq && workspace && (nseries == 0 || (x && psd)), "null buffer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  WelchParams p;
  p.x = x;
  p.inner = inner;
  p.outer_stride = outer_stride;
  p.sample_stride = sample_stride;
  p.nseries = nseries;
  p.S = w.S;
  p.K = w.K;
  p.Q = w.Q;
  p.nchunk = w.nchunk;
  p.N = w.N;
  p.M = w.M;
  p.P = w.P;
  p.logP = w.logP;
  p.G = w.G;
  p.bluestein = w.bluestein;
  p.fs = fs;
  p.window = window;
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  p.wscale = reinterpret_cast<double*>(ws);
  p.bhat = reinterpret_cast<const double2*>(ws + 16);
  p.part = reinterpret_cast<double*>(ws + welch_partial_offset(w));
  p.post = w.bluestein ? 0.25 / (static_cast<double>(w.P) * w.P) : 0.25;
  p.psd = psd;
  p.freq = freq;
  welch_prep_kernel<<<1, kWelchThreads, 0, s>>>(p);
  CU_CHECK(cudaGetLastError());
  if (nseries == 0) return B2INS_OK;
  const size_t fft_smem = static_cast<size_t>(w.P) * 24;
  const size_t smem = (static_cast<size_t>(w.G) * w.P + w.P / 2) * 16;
  if (w.bluestein) {   // K5's transform of the conjugate chirp: the forward transform runs K5's pipeline on conj z
    PsdFftParams f;
    std::memset(&f, 0, sizeof(f));
    f.N = w.N;
    f.M = w.M;
    f.P = w.P;
    f.logP = w.logP;
    f.bluestein = 1;
    f.bhat = reinterpret_cast<double2*>(ws + 16);
    CU_CHECK(cudaFuncSetAttribute(psd_chirp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 24));
    psd_chirp_kernel<<<1, kFftThreads, fft_smem, s>>>(f);
    CU_CHECK(cudaGetLastError());
  }
  // the bins a thread accumulates: 3 for transforms of at most 1024 points (several segments per CTA), else 17
  const bool small = w.P <= kWelchBatchPoints;
  void (*const fn)(WelchParams) =
      small ? (w.bluestein ? welch_kernel<kWelchAccSmall, true> : welch_kernel<kWelchAccSmall, false>)
            : (w.bluestein ? welch_kernel<kWelchAccLarge, true> : welch_kernel<kWelchAccLarge, false>);
  if (!small) CU_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 24));
  int per_sm = 1;
  CU_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kWelchThreads, smem));
  const int64_t items = nseries * w.nchunk;
  const int64_t cap = static_cast<int64_t>(sm_count()) * (per_sm > 0 ? per_sm : 1);
  fn<<<static_cast<unsigned>(items < cap ? items : cap), kWelchThreads, smem, s>>>(p);
  CU_CHECK(cudaGetLastError());
  if (w.nchunk > 1) {
    const int64_t total = nseries * (w.M + 1);
    welch_finish_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(p);
    CU_CHECK(cudaGetLastError());
  }
  return B2INS_OK;
}

int b2ins_welch_f64_host(double fs, int64_t n, int64_t nseries, const double* x, int64_t inner, int64_t outer_stride,
                         int64_t sample_stride, int64_t nperseg, int64_t noverlap, const double* window, double* psd,
                         double* freq) {
  WelchPlan w;
  const int chk = welch_check(fs, n, nseries, inner, outer_stride, sample_stride, nperseg, noverlap, &w);
  if (chk != B2INS_OK) return chk;
  ARG_CHECK(window && freq && (nseries == 0 || (x && psd)), "null buffer");
  const int64_t L = nperseg / 2 + 1;
  Staging st;
  const double* dx = st.in(x, series_elems(n, nseries, inner, outer_stride, sample_stride));
  const double* dw = st.in(window, nperseg);
  double* dpsd = st.out(psd, nseries * L);
  double* dfreq = st.out(freq, L);
  void* ws = st.scratch(b2ins_welch_workspace_bytes(n, nseries, nperseg, noverlap));
  return st.run([&](cudaStream_t s) {
    return b2ins_welch_f64(fs, n, nseries, dx, inner, outer_stride, sample_stride, nperseg, noverlap, dw, dpsd,
                           dfreq, ws, s);
  });
}

// ---------------------------------------------------------------- K1 plan ---
int b2ins_diag_noise_plan(double fs, int64_t runs, int64_t n, const b2ins_sensor_err* gyro_err,
                          const b2ins_sensor_err* accel_err, int sm_count_arg, double* coef, int64_t* plan) {
  return b2ins_diag_noise_plan_ex(fs, runs, n, gyro_err, accel_err, nullptr, nullptr, sm_count_arg, coef, plan);
}

int b2ins_diag_noise_plan_ex(double fs, int64_t runs, int64_t n, const b2ins_sensor_err* gyro_err,
                             const b2ins_sensor_err* accel_err, const b2ins_noise_terms* gyro_terms,
                             const b2ins_noise_terms* accel_terms, int sm_count_arg, double* coef, int64_t* plan) {
  ARG_CHECK(fs > 0.0, "fs must be positive");
  ARG_CHECK(runs > 0 && n > 0, "runs and n must be positive");
  ARG_CHECK(gyro_err && accel_err && coef && plan, "null buffer");
  NoiseModel m;
  const int rc = digest_noise(fs, runs, n, gyro_err, accel_err, gyro_terms, accel_terms, nullptr, nullptr, nullptr,
                              nullptr, &m);
  if (rc != B2INS_OK) return rc;
  NoiseParams& p = m.p;
  noise_plan(&p, sm_count_arg > 0 ? sm_count_arg : sm_count(), m.walk);
  for (int c = 0; c < 6; ++c) {
    const TriadNoise& e = (c < 3) ? p.accel : p.gyro;
    coef[c] = e.gm_a[c % 3];
    coef[6 + c] = e.gm_b[c % 3];
    coef[12 + c] = e.wd[c % 3];
  }
  plan[0] = p.nseg;
  plan[1] = p.seg_len;
  plan[2] = p.pass1_len;
  return B2INS_OK;
}

int64_t b2ins_psd_workspace_bytes(int64_t n, int64_t runs) {
  if (n <= 0 || runs <= 0) return 16;
  const int64_t L = psd_series_len(n) / 2 + 1;
  // (A, B) of every bin, then the transform of the chirp for the Bluestein lengths (<= 8192 complex)
  return runs * 3 * L * 2 * static_cast<int64_t>(sizeof(double)) + 8192 * 16 + 64;
}

int b2ins_psd_series_f64(double fs, int64_t n, int64_t runs, int sensor, int table_len,
                         const double* freq, const double* sxx3, uint64_t seed,
                         int64_t run_offset, double* series, void* workspace, void* stream) {
  ARG_CHECK(fs > 0.0 && n > 0 && runs >= 0, "bad fs/n/runs");
  ARG_CHECK(sensor == 0 || sensor == 1, "sensor must be 0 (accel) or 1 (gyro)");
  ARG_CHECK(table_len >= 2, "the PSD table needs at least two rows");
  if (runs == 0) return B2INS_OK;
  ARG_CHECK(freq && sxx3 && series && workspace, "null buffer");
  ARG_CHECK(runs * 3 <= 65535, "at most 21845 runs per call (grid.y)");
  PsdParams p;
  p.fs = fs;
  p.runs = runs;
  p.run_offset = run_offset;
  p.N = psd_series_len(n);
  p.L = p.N / 2 + 1;
  p.L0 = table_len;
  p.sensor = sensor;
  p.interp = (table_len != p.L) ? 1 : 0;  // time_series_from_psd.py:46
  p.k0 = static_cast<uint32_t>(seed);
  p.k1 = static_cast<uint32_t>(seed >> 32);
  p.freq = freq;
  p.sxx = sxx3;
  p.ab = static_cast<double*>(workspace);
  p.series = series;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  dim3 g1((p.L + kPsdThreads - 1) / kPsdThreads, static_cast<unsigned>(runs * 3));
  psd_phase_kernel<<<g1, kPsdThreads, 0, s>>>(p);
  int bluestein = 0;
  const int P = psd_direct_forced() ? 0 : psd_fft_plan(p.N, &bluestein);
  if (P == 0) {      // lengths without an FFT path: the O(N L) cosine synthesis
    dim3 g2((p.N + kPsdThreads - 1) / kPsdThreads, static_cast<unsigned>(runs * 3));
    psd_synth_kernel<<<g2, kPsdThreads, 0, s>>>(p);
    CU_CHECK(cudaGetLastError());
    return B2INS_OK;
  }
  PsdFftParams f;
  f.nseries = runs * 3;
  f.N = p.N;
  f.L = p.L;
  f.M = p.N / 2;
  f.P = P;
  f.logP = 0;
  while ((1 << f.logP) < P) ++f.logP;
  f.bluestein = bluestein;
  f.ab = p.ab;
  // the chirp transform sits behind the (A, B) block, 16-byte aligned
  uintptr_t tail = reinterpret_cast<uintptr_t>(p.ab + runs * 3 * static_cast<int64_t>(p.L) * 2);
  tail = (tail + 15) & ~static_cast<uintptr_t>(15);
  f.bhat = reinterpret_cast<double2*>(tail);
  f.series = series;
  const size_t smem = static_cast<size_t>(P) * 16 + static_cast<size_t>(P / 2) * 16;
  static int attr_dev = -1;
  int dev = 0;
  CU_CHECK(cudaGetDevice(&dev));
  if (attr_dev != dev) {
    CU_CHECK(cudaFuncSetAttribute(psd_fft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 24));
    CU_CHECK(cudaFuncSetAttribute(psd_chirp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 24));
    attr_dev = dev;
  }
  if (bluestein) psd_chirp_kernel<<<1, kFftThreads, smem, s>>>(f);
  const int64_t grid = f.nseries < 2 * sm_count() ? f.nseries : 2 * sm_count();
  psd_fft_kernel<<<static_cast<unsigned>(grid), kFftThreads, smem, s>>>(f);
  CU_CHECK(cudaGetLastError());
  return B2INS_OK;
}

// ---------------------------------------------------------------- host ------
int64_t b2ins_path_rows(const double* motion_def, int64_t segs, double fs) {
  if (!motion_def || segs <= 0 || !(fs > 0.0)) return -1;
  return b2ins_host::path_rows(motion_def, segs, fs);
}

int64_t b2ins_path_gen_ex_host(const double* ini, const double* motion_def, int64_t segs, double fs,
                               double osr, double fs_gps, double fs_odo, const double* mobility,
                               int ref_frame, int64_t cap, double* imu, double* nav, double* gps,
                               int64_t* gps_rows, double* odo, const double* geomag_n, double* mag) {
  if (!ini || !motion_def || !mobility || !imu || !nav || segs <= 0 || !(fs > 0.0) || !(osr >= 1.0) ||
      (ref_frame != 0 && ref_frame != 1) || (gps && !(fs_gps > 0.0)) || (geomag_n && !mag)) {
    fail(B2INS_ERR_ARG, "bad argument to b2ins_path_gen_host");
    return -1;
  }
  return b2ins_host::path_gen(ini, motion_def, segs, fs, osr, fs_gps, fs_odo, mobility, ref_frame,
                              cap, imu, nav, gps, gps_rows, odo, geomag_n, geomag_n ? mag : nullptr);
}

int64_t b2ins_path_gen_host(const double* ini, const double* motion_def, int64_t segs, double fs,
                            double osr, double fs_gps, double fs_odo, const double* mobility,
                            int ref_frame, int64_t cap, double* imu, double* nav, double* gps,
                            int64_t* gps_rows, double* odo) {
  return b2ins_path_gen_ex_host(ini, motion_def, segs, fs, osr, fs_gps, fs_odo, mobility, ref_frame,
                                cap, imu, nav, gps, gps_rows, odo, nullptr, nullptr);
}

// ---------------------------------------------------------------- diag ------
__global__ void dfma_rate_kernel(double* out, int iters) {
  double a0 = threadIdx.x * 1e-9, a1 = a0 + 1, a2 = a0 + 2, a3 = a0 + 3, a4 = a0 + 4,
         a5 = a0 + 5, a6 = a0 + 6, a7 = a0 + 7;
  const double m = 1.0000001, c = 1e-9;
  for (int i = 0; i < iters; ++i) {
    a0 = fma(a0, m, c); a1 = fma(a1, m, c); a2 = fma(a2, m, c); a3 = fma(a3, m, c);
    a4 = fma(a4, m, c); a5 = fma(a5, m, c); a6 = fma(a6, m, c); a7 = fma(a7, m, c);
  }
  out[static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

int b2ins_diag_auto_lanes(int64_t runs, int fused, int sm_count_arg) {
  return auto_lanes(runs < 1 ? 1 : runs, fused != 0, sm_count_arg);
}

int b2ins_diag_mc_shape(int lanes_per_run, int ref_frame, int* shape3) {
  ARG_CHECK(shape3, "null output");
  ARG_CHECK(lanes_per_run == 1 || lanes_per_run == 2 || lanes_per_run == 4 || lanes_per_run == 8 ||
                lanes_per_run == 16 || lanes_per_run == 32, "lanes_per_run must be 1,2,4,8,16 or 32");
  McShape sh = default_shape(lanes_per_run, ref_frame);
  shape_override(&sh);   // (G = 1 launches of 2^18 runs and more take the single-warp form whatever this says)
  shape3[0] = sh.spec ? sh.P : 0;
  shape3[1] = sh.spec ? sh.WI : 0;
  shape3[2] = (sh.spec && sh.split) ? 1 : 0;
  return B2INS_OK;
}

int b2ins_diag_dfma_rate(double* dfma_per_s) {
  ARG_CHECK(dfma_per_s, "null output");
  const int blocks = sm_count() * 8, threads = 256, iters = 8000;
  DevBuf out;
  CU_CHECK(out.alloc(sizeof(double) * blocks * threads));
  cudaEvent_t e0, e1;
  CU_CHECK(cudaEventCreate(&e0));
  CU_CHECK(cudaEventCreate(&e1));
  float best = 1e30f;
  for (int rep = 0; rep < 4; ++rep) {  // rep 0 warms up
    CU_CHECK(cudaEventRecord(e0, nullptr));
    dfma_rate_kernel<<<blocks, threads>>>(out.d(), iters);
    CU_CHECK(cudaEventRecord(e1, nullptr));
    CU_CHECK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CU_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *dfma_per_s = static_cast<double>(blocks) * threads * iters * 8.0 / (best * 1e-3);
  return B2INS_OK;
}

}  // extern "C"

// The production FP64 primitives and the noise generator, elementwise, so that the suite measures them
// as the device runs them (tests/test_gpu_fastmath.py).  One instantiation per function: each body is
// the inlined production function and nothing else.
template <int FN>
__global__ void fastmath_diag_kernel(int64_t n, const double* __restrict__ a, const double* __restrict__ b,
                                     double* __restrict__ out0, double* __restrict__ out1) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const double x = a[i];
    double s = 0.0, c = 0.0;
    if (FN == B2INS_FM_RCP) s = rcp_nr(x);
    if (FN == B2INS_FM_DIV) s = div_nr(x, b[i]);
    if (FN == B2INS_FM_SQRT) s = sqrt_nr(x);
    if (FN == B2INS_FM_RSQRT) s = rsqrt_nr(x);
    if (FN == B2INS_FM_SINCOS) sincos_bounded(x, &s, &c);
    if (FN == B2INS_FM_SINCOS_ANGLE) sincos_angle(x, &s, &c);
    if (FN == B2INS_FM_SINCOSPI) sincospi_2u(x, &s, &c);
    if (FN == B2INS_FM_LOG) s = log_unit(x);
    out0[i] = s;
    if (out1) out1[i] = c;
  }
}

__global__ void philox_diag_kernel(int64_t n, const uint32_t* __restrict__ ck, uint32_t* __restrict__ words) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint32_t* c = ck + 6 * i;
    const PhiloxOut x = philox4x32_10(c[0], c[1], c[2], c[3], c[4], c[5]);
    words[4 * i] = x.x0;
    words[4 * i + 1] = x.x1;
    words[4 * i + 2] = x.x2;
    words[4 * i + 3] = x.x3;
  }
}

__global__ void normal_diag_kernel(int64_t n, const uint32_t* __restrict__ words, double* __restrict__ z) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint32_t* w = words + 4 * i;
    const Normal2 p = normal_from_words(PhiloxOut{w[0], w[1], w[2], w[3]});
    z[2 * i] = p.z0;
    z[2 * i + 1] = p.z1;
  }
}

static unsigned diag_grid(int64_t n) {
  const int64_t cap = 32 * static_cast<int64_t>(sm_count());
  const int64_t g = (n + 255) / 256;
  return static_cast<unsigned>(g < cap ? g : cap);
}

extern "C" {

int b2ins_diag_fastmath_f64(int fn, int64_t n, const double* a, const double* b, double* out0, double* out1) {
  ARG_CHECK(fn >= B2INS_FM_RCP && fn <= B2INS_FM_LOG, "unknown function %d", fn);
  ARG_CHECK(n >= 0, "bad n");
  if (n == 0) return B2INS_OK;
  const bool pair = fn == B2INS_FM_SINCOS || fn == B2INS_FM_SINCOS_ANGLE || fn == B2INS_FM_SINCOSPI;
  ARG_CHECK(a && out0 && (fn != B2INS_FM_DIV || b) && (!pair || out1), "null buffer");
  const unsigned g = diag_grid(n);
  switch (fn) {
    case B2INS_FM_RCP: fastmath_diag_kernel<B2INS_FM_RCP><<<g, 256>>>(n, a, b, out0, nullptr); break;
    case B2INS_FM_DIV: fastmath_diag_kernel<B2INS_FM_DIV><<<g, 256>>>(n, a, b, out0, nullptr); break;
    case B2INS_FM_SQRT: fastmath_diag_kernel<B2INS_FM_SQRT><<<g, 256>>>(n, a, b, out0, nullptr); break;
    case B2INS_FM_RSQRT: fastmath_diag_kernel<B2INS_FM_RSQRT><<<g, 256>>>(n, a, b, out0, nullptr); break;
    case B2INS_FM_SINCOS: fastmath_diag_kernel<B2INS_FM_SINCOS><<<g, 256>>>(n, a, b, out0, out1); break;
    case B2INS_FM_SINCOS_ANGLE:
      fastmath_diag_kernel<B2INS_FM_SINCOS_ANGLE><<<g, 256>>>(n, a, b, out0, out1);
      break;
    case B2INS_FM_SINCOSPI: fastmath_diag_kernel<B2INS_FM_SINCOSPI><<<g, 256>>>(n, a, b, out0, out1); break;
    default: fastmath_diag_kernel<B2INS_FM_LOG><<<g, 256>>>(n, a, b, out0, nullptr); break;
  }
  CU_CHECK(cudaGetLastError());
  CU_CHECK(cudaDeviceSynchronize());
  return B2INS_OK;
}

int b2ins_diag_philox(int64_t n, const uint32_t* ctr_key, uint32_t* words) {
  ARG_CHECK(n >= 0, "bad n");
  if (n == 0) return B2INS_OK;
  ARG_CHECK(ctr_key && words, "null buffer");
  philox_diag_kernel<<<diag_grid(n), 256>>>(n, ctr_key, words);
  CU_CHECK(cudaGetLastError());
  CU_CHECK(cudaDeviceSynchronize());
  return B2INS_OK;
}

int b2ins_diag_normal_from_words(int64_t n, const uint32_t* words, double* z) {
  ARG_CHECK(n >= 0, "bad n");
  if (n == 0) return B2INS_OK;
  ARG_CHECK(words && z, "null buffer");
  normal_diag_kernel<<<diag_grid(n), 256>>>(n, words, z);
  CU_CHECK(cudaGetLastError());
  CU_CHECK(cudaDeviceSynchronize());
  return B2INS_OK;
}

#ifdef B2INS_PHASE_CLOCKS
// tools only: the kPhaseClocks cumulative warp-cycle counters (slots: mc_kernel.cuh, mc_spec_kernel.cuh,
// mc_av_kernel.cuh)
int b2ins_diag_phase_clocks(unsigned long long* out16, int reset) {
  if (out16) cudaMemcpyFromSymbol(out16, g_phase_clocks, sizeof(unsigned long long) * kPhaseClocks);
  if (reset) {
    unsigned long long z[kPhaseClocks] = {};
    cudaMemcpyToSymbol(g_phase_clocks, z, sizeof(z));
  }
  return B2INS_OK;
}
#endif

}  // extern "C"
