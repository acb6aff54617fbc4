// Instantiations of the warp-specialised Monte-Carlo kernel for ONE reference frame (B2_RF), see
// internal.h.  The shapes: four-warp CTAs (every warp on its own SM sub-partition) with three
// producers, eight-warp CTAs with six producers and a spare warp, the paired layout for wide groups.
#include "internal.h"
#include "mc_spec_kernel.cuh"
#include "mc_av_kernel.cuh"

namespace b2ins {
#ifndef B2INS_MC_SPEC_HELPERS   // (b2ins_api.cu includes this file once per frame under B2INS_SINGLE_TU)
#define B2INS_MC_SPEC_HELPERS
namespace {

template <int G, int RF, int P, int WI, bool SPLIT, int MINB>
void launch_one(const McParams& p, cudaStream_t s) {
  const int64_t runs_per_cta = static_cast<int64_t>(WI) * (32 / G);
  const unsigned grid = static_cast<unsigned>((p.runs + runs_per_cta - 1) / runs_per_cta);
  mc_spec_kernel<G, RF, P, WI, SPLIT, MINB><<<grid, SpecShape<G, P, WI>::kThreads, 0, s>>>(p);
}

// the step split over an attitude and a velocity warp (ref_frame 1 only): shape "6,2,0"
template <int G>
void launch_av(const McParams& p, cudaStream_t s) {
  const int64_t runs_per_cta = 32 / G;
  const unsigned grid = static_cast<unsigned>((p.runs + runs_per_cta - 1) / runs_per_cta);
  mc_av_kernel<G><<<grid, AvShape<G>::kWarps * 32, 0, s>>>(p);
}

}  // namespace
#endif

bool B2_SPEC_NAME(const McParams& p, const McShape& sh, cudaStream_t s) {
  const int key = sh.G * 1000 + sh.P * 100 + sh.WI * 10 + (sh.split ? 1 : 0);
  switch (key) {
    case 1310: launch_one<1, B2_RF, 3, 1, false, 3>(p, s); return true;
    case 1610: launch_one<1, B2_RF, 6, 1, false, 2>(p, s); return true;
    case 2310: launch_one<2, B2_RF, 3, 1, false, 3>(p, s); return true;
    case 2610: launch_one<2, B2_RF, 6, 1, false, 2>(p, s); return true;
    case 4310: launch_one<4, B2_RF, 3, 1, false, 2>(p, s); return true;
    case 4311: launch_one<4, B2_RF, 3, 1, true, 2>(p, s); return true;
    case 4610: launch_one<4, B2_RF, 6, 1, false, 1>(p, s); return true;
    case 4611: launch_one<4, B2_RF, 6, 1, true, 1>(p, s); return true;
#if B2_RF == 1
    case 4620: launch_av<4>(p, s); return true;
    case 8620: launch_av<8>(p, s); return true;
#endif
    case 8120: launch_one<8, B2_RF, 1, 2, false, 2>(p, s); return true;
    case 8610: launch_one<8, B2_RF, 6, 1, false, 1>(p, s); return true;
    case 16140: launch_one<16, B2_RF, 1, 4, false, 1>(p, s); return true;
    case 16141: launch_one<16, B2_RF, 1, 4, true, 1>(p, s); return true;
    case 32141: launch_one<32, B2_RF, 1, 4, true, 1>(p, s); return true;
    default: return false;
  }
}

}  // namespace b2ins
