// seaweedfs_b200/csrc/kernels.h — host-callable launchers of the sm_90a kernels (kernels.cu).
#pragma once
#include <cuda_runtime.h>

#include <atomic>

#include "apply_params.h"

namespace swec {

extern std::atomic<unsigned long long> g_kernel_launches;

// tuning knobs: launch shape of the Horner kernels (swec_set_option / SWEC_ENC_THREADS, SWEC_ENC_UNROLL,
// SWEC_CTAS_PER_SM).  ctas_per_sm = resident CTAs per SM the persistent grids are sized for.
extern std::atomic<long> g_opt_enc_threads, g_opt_enc_unroll, g_opt_ctas_per_sm;
// measurement knobs: xtime instruction-mix variant of run-time specialised kernels (device_common.cuh), and
// whether RS(10,4) encode takes the ahead-of-time kernel (1) or is specialised at run time like any matrix (0)
extern std::atomic<long> g_opt_xt_variant, g_opt_use_aot;
// measurement knob: run-time specialised kernels are generated with shared power chains (codegen.h share_powers): fewer
// multiply-by-2 steps (RS(10,4) encode 24 -> 20, worst-case decode 27 -> 21); bytes checked on the GPU
// (tests/test_kernel_variants.py), speed not yet measured.  Part of the specialised kernel's cache key (jit.cc)
extern std::atomic<long> g_opt_jit_share_powers;
// Power policy (kernels.cu).  A GPU that encodes back to back for more than a few hundred ms can run into its power
// cap and lower the SM clock; from then on the 4-instruction multiply-by-2 step (variant 2: fewer instructions, far
// fewer IMADs) can be FASTER than the 5-instruction one that wins while the GPU still boosts.  "power_mode": 0 = auto (low-power once the
// Horner kernels own > 45 % of the device's last second), 1 = always the boost-clock variant (default), 2 = always the low-power variant.
extern std::atomic<long> g_opt_power_mode;
void note_kernel_work(double est_ms);   // called by every Horner launch: feeds the auto policy
double power_heat_ms();                 // Horner-kernel milliseconds of the last ~second on the current device (decayed)
bool low_power_now();                   // which variant the next Horner launch on the current device takes
int effective_xt_variant();             // variant for run-time specialised kernels (explicit xt_variant wins)
int encode_ctas_per_sm();

cudaError_t launch_rs10x4_encode(const SwecApplyParams& p, bool blocked, cudaStream_t s);
// aot_recon.cu: reconstruct matrices compiled with the library (every single-shard loss of RS(10,4) + the worst case)
int aot_recon_find(int r, int k, const unsigned char* coef);  // index or -1
int aot_recon_count();
unsigned long long aot_recon_launches();  // launches of those kernels by this process
cudaError_t launch_aot_recon(int idx, const SwecApplyParams& p, cudaStream_t s);  // flat layout
// replicated_tables: [K][2][16][32] words (lane-replicated), device memory, 16-byte aligned
cudaError_t launch_table_apply(const SwecApplyParams& p, const u32* replicated_tables, int K, int r, cudaStream_t s);
// compact_tables: [K][2][16] words, device memory
cudaError_t launch_bytes_apply(const SwecApplyParams& p, const u32* compact_tables, int K, int r, u64 nbytes,
                               cudaStream_t s);
cudaError_t launch_synth(void* dst, u64 byte_offset, u64 nbytes, u64 seed, cudaStream_t s);
cudaError_t launch_digest(const void* src, u64 nbytes, u64* out_dev, cudaStream_t s);
cudaError_t launch_compare(const void* a, const void* b, u64 nbytes, unsigned long long* out_dev, cudaStream_t s);

}  // namespace swec
