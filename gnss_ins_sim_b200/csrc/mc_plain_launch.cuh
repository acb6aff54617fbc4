// Instantiations of the single-warp Monte-Carlo kernel for ONE reference frame (B2_RF), see internal.h.
#include "internal.h"

namespace b2ins {
#ifndef B2INS_MC_PLAIN_HELPERS   // (b2ins_api.cu includes this file once per frame under B2INS_SINGLE_TU)
#define B2INS_MC_PLAIN_HELPERS
namespace {

template <int G, int RF>
void launch_g(const McParams& p, bool fed, bool proc, cudaStream_t s) {
  const int64_t runs_per_cta = static_cast<int64_t>(kWarps) * (32 / G);
  const unsigned grid = static_cast<unsigned>((p.runs + runs_per_cta - 1) / runs_per_cta);
  if (fed) {
    if (proc)
      mc_kernel<G, RF, true, true><<<grid, kThreads, 0, s>>>(p);
    else
      mc_kernel<G, RF, true, false><<<grid, kThreads, 0, s>>>(p);
  } else {
    if (proc)
      mc_kernel<G, RF, false, true><<<grid, kThreads, 0, s>>>(p);
    else
      mc_kernel<G, RF, false, false><<<grid, kThreads, 0, s>>>(p);
  }
}

}  // namespace
#endif

void B2_PLAIN_NAME(const McParams& p, int lanes, bool fed, bool proc, cudaStream_t s) {
  switch (lanes) {
    case 1: launch_g<1, B2_RF>(p, fed, proc, s); break;
    case 2: launch_g<2, B2_RF>(p, fed, proc, s); break;
    case 4: launch_g<4, B2_RF>(p, fed, proc, s); break;
    case 8: launch_g<8, B2_RF>(p, fed, proc, s); break;
    case 16: launch_g<16, B2_RF>(p, fed, proc, s); break;
    default: launch_g<32, B2_RF>(p, fed, proc, s); break;
  }
}

}  // namespace b2ins
