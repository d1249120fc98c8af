// seaweedfs_b200/csrc/aot_recon.cu — ahead-of-time Horner kernels for the reconstruct matrices a volume server
// meets first: every single-shard loss of RS(10,4) (ec.rebuild after one disk/server died, and every degraded
// read behind it: enc.Reconstruct / ReconstructData, weed/storage/erasure_coding/ec_encoder.go:360,
// weed/storage/store_ec.go:551) and the worst case, data shards 0-3 lost (BASELINE configs[2]).
//
// The reference keeps decode matrices in an LRU (seaweed-volume/vendor/reed-solomon-erasure/src/core.rs:25,700-734);
// here the "matrix" is a kernel.  These 15 are compiled with the library, so they cost nothing at run time, need no
// NVRTC, and serve streams of ANY length (no warm-up threshold).  All other patterns are specialised at run time
// and kept in the on-disk cubin cache (jit.cc).  The combiners come from the same generator as the encode kernel
// (codegen_main.cc --aot-recon 10 4); both multiply-by-2 spellings are compiled, like the encode kernel.
#include <cuda_runtime.h>

#include <atomic>
#include <cstring>

#ifndef SWEC_XT_VARIANT
#define SWEC_XT_VARIANT 0
#endif
#include "device_common.cuh"

namespace swec_aot_boost {
#include "gen_aot_recon.inc"
}
#undef SWEC_XT1A
#undef SWEC_XT1B
#define SWEC_XT1A(a, s) swec_xt1_v<2>((a), (s))
#define SWEC_XT1B(a, s) swec_xt1_v<2>((a), (s))
namespace swec_aot_lowpower {
#include "gen_aot_recon.inc"
}
#undef SWEC_XT1A
#undef SWEC_XT1B
#define SWEC_XT1A(a, s) swec_xt1_v<SWEC_XT_VARIANT>((a), (s))
#define SWEC_XT1B(a, s) swec_xt1_v<SWEC_XT_VARIANT>((a), (s))
#include "gen_aot_recon_keys.inc"
#include "kernels.h"

namespace swec {

constexpr int kAotThreads = 512, kAotUnroll = 2;  // the measured-best shape of the encode kernel (DESIGN.md §6)

// flat layout only: reconstruct works on whole shard streams (the blocked layout is the .dat striping, an encode matter)
template <class Combiner>
__global__ void __launch_bounds__(kAotThreads) swec_aot_recon(const __grid_constant__ SwecApplyParams p) {
    swec_horner_body<Combiner, false, kAotUnroll>(p);
}

int aot_recon_find(int r, int k, const unsigned char* coef) {
    for (int i = 0; i < SWEC_AOT_RECON_COUNT; i++)
        if (kAotReconKeys[i].r == r && kAotReconKeys[i].k == k && memcmp(kAotReconKeys[i].c, coef, size_t(r) * size_t(k)) == 0)
            return i;
    return -1;
}

int aot_recon_count() { return SWEC_AOT_RECON_COUNT; }

static std::atomic<unsigned long long> g_aot_launches{0};
unsigned long long aot_recon_launches() { return g_aot_launches.load(); }

cudaError_t launch_aot_recon(int idx, const SwecApplyParams& p, cudaStream_t s) {
    if (p.nvec == 0) return cudaSuccess;
    if (idx < 0 || idx >= SWEC_AOT_RECON_COUNT) return cudaErrorInvalidValue;
    // light kernels (one output row: few registers) fit two CTAs per SM; the 4-row worst case one, like encode
    const unsigned grid = grid_for(p.nvec, u64(kAotThreads) * kAotUnroll, kAotReconKeys[idx].r >= 3 ? 1 : 2);
    const bool lp = low_power_now();
    note_kernel_work(double(p.nvec) * 16.0 * double(kAotReconKeys[idx].k + kAotReconKeys[idx].r) / 3.0e12 * 1e3);
    g_aot_launches++;
    switch (idx) {
#define SWEC_AOT_CASE(I)                                                                              \
    case I:                                                                                           \
        if (lp) swec_aot_recon<swec_aot_lowpower::SwecAotRecon##I><<<grid, kAotThreads, 0, s>>>(p);     \
        else swec_aot_recon<swec_aot_boost::SwecAotRecon##I><<<grid, kAotThreads, 0, s>>>(p);           \
        break;
        SWEC_AOT_RECON_FOREACH(SWEC_AOT_CASE)
#undef SWEC_AOT_CASE
        default: return cudaErrorInvalidValue;
    }
    return launched();
}

}  // namespace swec
