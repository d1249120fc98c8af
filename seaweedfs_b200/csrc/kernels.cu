// seaweedfs_b200/csrc/kernels.cu — ahead-of-time sm_90a kernels and their launchers.
//
//   rs10x4_encode_{flat,blocked}  RS(10,4) parity generation, constant matrix compiled in
//                                 (replaces enc.Encode, weed/storage/erasure_coding/ec_encoder.go:265)
//   swec_table_kernel             any R≤4 × K≤32 run-time matrix through 4-bit split multiply
//                                 tables in shared memory, tables fetched with one TMA bulk copy
//                                 (replaces enc.Reconstruct / ReconstructData for cold matrices,
//                                 ec_encoder.go:360, weed/storage/store_ec.go:551)
//   swec_bytes_kernel             byte-granular fallback for unaligned pointers and <16 B tails
//   swec_synth_kernel             counter-based synthetic volume bytes (measurement only)
//   swec_digest_kernel            64-bit order-sensitive digest of a buffer (measurement only)
//   swec_compare_kernel           count of differing 16-byte vectors (parity verify / scrub)
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>

#ifndef SWEC_XT_VARIANT
#define SWEC_XT_VARIANT 0
#endif
#include "device_common.cuh"
#include "tma_fetch.cuh"
#include "gen_rs10x4_encode.inc"
// the same combiner once more with the low-power step (variant 2) bound to both spellings
#undef SWEC_XT1A
#undef SWEC_XT1B
#define SWEC_XT1A(a, s) swec_xt1_v<2>((a), (s))
#define SWEC_XT1B(a, s) swec_xt1_v<2>((a), (s))
#include "gen_rs10x4_encode_lp.inc"
#undef SWEC_XT1A
#undef SWEC_XT1B
#define SWEC_XT1A(a, s) swec_xt1_v<SWEC_XT_VARIANT>((a), (s))
#define SWEC_XT1B(a, s) swec_xt1_v<SWEC_XT_VARIANT>((a), (s))
#include "kernels.h"

#include <chrono>
#include <cmath>
#include <mutex>

namespace swec {

std::atomic<unsigned long long> g_kernel_launches{0};

// ------------------------------------------------------------------ RS(10,4) encode, AOT Horner

// Launch shape is a tuning surface (threads per CTA × column slices per thread); the default is the
// measured best (DESIGN.md §6), SWEC_ENC_THREADS / SWEC_ENC_UNROLL select the others for sweeps.
template <int THREADS, int UNROLL, bool BLOCKED, bool LOW_POWER = false>
__global__ void __launch_bounds__(THREADS) rs10x4_encode(const __grid_constant__ SwecApplyParams p) {
    if (LOW_POWER) swec_horner_body<Rs10x4EncodeLP, BLOCKED, UNROLL>(p);
    else swec_horner_body<Rs10x4Encode, BLOCKED, UNROLL>(p);
}

// ------------------------------------------------------------------ run-time matrix, smem tables
// Table word for input i, nibble half h (0 = low, 1 = high), nibble value v packs the contribution
// to the (up to) four outputs: byte p = M[p][i] ⊗ (v << 4h).  Each entry is replicated once per
// lane — word index ((i*2+h)*16+v)*32+lane — so lane l always hits bank l: conflict-free no matter
// what the data bytes are.  K*4 KiB per CTA, fetched by one cp.async.bulk (TMA, SASS UBLKCP).

template <int KT>  // KT > 0: inputs known at compile time (loads hoisted); 0: run-time loop
__global__ void __launch_bounds__(256) swec_table_kernel(const __grid_constant__ SwecApplyParams p,
                                                          const u32* __restrict__ tables, int k_rt, int r) {
    extern __shared__ __align__(128) u32 tab[];
    __shared__ __align__(8) u64 mbar;
    const int K = KT > 0 ? KT : k_rt;
    tma_fetch(tab, tables, (u32)K * 4096u, &mbar);
    const u32 lane4 = (threadIdx.x & 31u) * 4u;
    const char* tb = reinterpret_cast<const char*>(tab);
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 v = (u64)blockIdx.x * blockDim.x + threadIdx.x; v < p.nvec; v += stride) {
        const u64 off = v << 4;
        u32 acc[16];
#pragma unroll
        for (int j = 0; j < 16; j++) acc[j] = 0;
        auto fold = [&](int i, const uint4& d) {
            const char* t = tb + (u32)i * 4096u + lane4;  // low table; high table 2048 bytes further
            const u32 w[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
            for (int c = 0; c < 4; c++) {
#pragma unroll
                for (int b = 0; b < 4; b++) {
                    const u32 byte = (w[c] >> (8 * b)) & 0xffu;
                    const u32 lo = *reinterpret_cast<const u32*>(t + ((byte & 15u) << 7));
                    const u32 hi = *reinterpret_cast<const u32*>(t + 2048 + ((byte >> 4) << 7));
                    acc[c * 4 + b] = swec_x3(acc[c * 4 + b], lo, hi);
                }
            }
        };
        if (KT > 0) {
            uint4 d[KT > 0 ? KT : 1];
#pragma unroll
            for (int i = 0; i < KT; i++) d[i] = swec_ldg_stream(p.in[i] + off);
#pragma unroll
            for (int i = 0; i < KT; i++) fold(i, d[i]);
        } else {
            int i = 0;
            for (; i + 2 <= K; i += 2) {
                const uint4 d0 = swec_ldg_stream(p.in[i] + off);
                const uint4 d1 = swec_ldg_stream(p.in[i + 1] + off);
                fold(i, d0);
                fold(i + 1, d1);
            }
            if (i < K) fold(i, swec_ldg_stream(p.in[i] + off));
        }
        // acc[c*4+b] holds the r output bytes of column 16v+4c+b; regroup into one word per output
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (q < r) {
                uint4 o;
                u32* ow = reinterpret_cast<u32*>(&o);
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const u32 lo2 = __byte_perm(acc[c * 4 + 0], acc[c * 4 + 1], 0x0040 + q * 0x0011);
                    const u32 hi2 = __byte_perm(acc[c * 4 + 2], acc[c * 4 + 3], 0x0040 + q * 0x0011);
                    ow[c] = __byte_perm(lo2, hi2, 0x5410);
                }
                swec_stg_stream(p.out[q] + off, o);
            }
        }
    }
}

// Byte-granular fallback: any alignment, any length.  Tables are the compact (un-replicated)
// [K][2][16] words in global memory (L1-resident).
__global__ void __launch_bounds__(256) swec_bytes_kernel(const __grid_constant__ SwecApplyParams p,
                                                          const u32* __restrict__ compact, int K, int r,
                                                          u64 nbytes) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 x = (u64)blockIdx.x * blockDim.x + threadIdx.x; x < nbytes; x += stride) {
        u32 acc = 0;
        for (int i = 0; i < K; i++) {
            const u32 byte = p.in[i][x];
            acc ^= __ldg(&compact[i * 32 + (byte & 15u)]) ^ __ldg(&compact[i * 32 + 16 + (byte >> 4)]);
        }
        for (int q = 0; q < r; q++) p.out[q][x] = (u8)(acc >> (8 * q));
    }
}

// ------------------------------------------------------------------ measurement helpers

__device__ __forceinline__ u64 splitmix64_at(u64 seed, u64 j) {
    u64 z = seed + (j + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// dst[0..n) = bytes [byte_offset, byte_offset+n) of the seeded stream; byte_offset and n multiples of 8
__global__ void __launch_bounds__(256) swec_synth_kernel(u64* __restrict__ dst, u64 first_word, u64 nwords, u64 seed) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < nwords; j += stride)
        dst[j] = splitmix64_at(seed, first_word + j);
}

// digest = Σ_j mix(word_j + j·odd) (mod 2^64) over 8-byte words; tail bytes zero-padded.
__global__ void __launch_bounds__(256) swec_digest_kernel(const u8* __restrict__ src, u64 nbytes, u64* __restrict__ out) {
    const u64 nwords = (nbytes + 7) >> 3;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    u64 sum = 0;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < nwords; j += stride) {
        u64 w;
        if ((j + 1) * 8 <= nbytes && (reinterpret_cast<unsigned long long>(src) & 7) == 0) {
            w = reinterpret_cast<const u64*>(src)[j];
        } else {
            w = 0;
            for (int b = 0; b < 8; b++)
                if (j * 8 + b < nbytes) w |= (u64)src[j * 8 + b] << (8 * b);
        }
        sum += splitmix64_at(w, j);
    }
    for (int s = 16; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
    if ((threadIdx.x & 31) == 0) atomicAdd(reinterpret_cast<unsigned long long*>(out), sum);
}

// counts 16-byte vectors where a != b; a partial last vector (nbytes % 16 bytes) is one vector, as is every vector of
// an unaligned pair, which is compared byte by byte
__global__ void __launch_bounds__(256) swec_compare_kernel(const u8* __restrict__ a, const u8* __restrict__ b,
                                                            u64 nbytes, unsigned long long* __restrict__ mismatches) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const bool aligned = ((reinterpret_cast<unsigned long long>(a) | reinterpret_cast<unsigned long long>(b)) & 15) == 0;
    const u64 nvec = (nbytes + 15) >> 4;
    unsigned long long bad = 0;
    for (u64 v = (u64)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
        const u64 off = v << 4;
        if (aligned && off + 16 <= nbytes) {
            const uint4 x = swec_ldg_stream(a + off), y = swec_ldg_stream(b + off);
            bad += ((x.x ^ y.x) | (x.y ^ y.y) | (x.z ^ y.z) | (x.w ^ y.w)) != 0;
        } else {
            bool diff = false;
            for (u64 x = off; x < nbytes && x < off + 16; x++) diff |= a[x] != b[x];
            bad += diff;
        }
    }
    if (bad) atomicAdd(mismatches, bad);
}

// ------------------------------------------------------------------ launchers

int sm_count() {
    static std::atomic<int> cached[64];  // 0: not asked yet
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return 132;
    int n = cached[dev].load(std::memory_order_relaxed);
    if (!n) {
        n = 132;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        cached[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}

unsigned grid_cap(u64 need, int ctas_per_sm) {
    return unsigned(std::max<u64>(1, std::min<u64>(need, u64(sm_count()) * u64(ctas_per_sm))));
}

// ---- tuning options (defaults = measured best, DESIGN.md §6); env at start-up, swec_set_option later
static long env_long(const char* name, long dflt) {
    const char* e = getenv(name);
    return e && *e ? atol(e) : dflt;
}
std::atomic<long> g_opt_enc_threads{env_long("SWEC_ENC_THREADS", 512)};
std::atomic<long> g_opt_enc_unroll{env_long("SWEC_ENC_UNROLL", 2)};
std::atomic<long> g_opt_ctas_per_sm{env_long("SWEC_CTAS_PER_SM", 0)};  // 0 = derive from the shape
std::atomic<long> g_opt_xt_variant{env_long("SWEC_XT_VARIANT_JIT", SWEC_XT_VARIANT)};
std::atomic<long> g_opt_use_aot{env_long("SWEC_USE_AOT", 1)};
std::atomic<long> g_opt_jit_share_powers{env_long("SWEC_JIT_SHARE_POWERS", 0)};
std::atomic<long> g_opt_power_mode{env_long("SWEC_POWER_MODE", 1)};

// ---- power policy: "heat" = kernel milliseconds recently spent on the device, decaying with a 1 s time
// constant.  Continuous encoding drives it towards 1000 x duty cycle; a 13-launch burst leaves it below 100.
// On a GPU that reaches its power cap under sustained encoding, the low-power variant (fewer instructions per step) is
// the faster one once the clock has dropped, the boost variant while the GPU still boosts.  Auto switches at 450 ms of
// kernel time in the last second and keeps the boost variant for bursts and for batches with other kernels in between.
// It is not the default: on an H100 SXM at 700 W the clock stays at 1,980 MHz under sustained encoding, and the
// low-power variant is the slower one there (15.96 vs 15.36 ms per 30 GiB volume in bench.py's `sustained` leg).
namespace {
struct Heat {
    std::mutex mu;
    double level = 0;
    std::chrono::steady_clock::time_point last{};
};
Heat g_heat[64];
constexpr double kHeatTauMs = 1000.0, kHeatHotMs = 450.0;  // hot = the Horner kernels own > 45 % of the last second:
// from cold that is ~0.6 s of back-to-back launches
Heat& heat_here() {
    int dev = 0;
    cudaGetDevice(&dev);
    return g_heat[(dev >= 0 && dev < 64) ? dev : 0];
}
double decayed(Heat& h, std::chrono::steady_clock::time_point now) {
    if (h.last.time_since_epoch().count() == 0) return 0;
    const double dt = std::chrono::duration<double, std::milli>(now - h.last).count();
    return h.level * std::exp(-dt / kHeatTauMs);
}
}  // namespace

void note_kernel_work(double est_ms) {
    Heat& h = heat_here();
    const auto now = std::chrono::steady_clock::now();
    std::lock_guard<std::mutex> lk(h.mu);
    h.level = decayed(h, now) + est_ms;
    h.last = now;
}

bool low_power_now() {
    const long mode = g_opt_power_mode.load();
    if (mode == 1) return false;
    if (mode == 2) return true;
    Heat& h = heat_here();
    const auto now = std::chrono::steady_clock::now();
    std::lock_guard<std::mutex> lk(h.mu);
    const double level = decayed(h, now);
    static const bool debug = getenv("SWEC_DEBUG_POWER") != nullptr;
    if (debug) fprintf(stderr, "[swec] power policy: heat %.1f ms (hot above %.0f) -> %s variant\n", level, kHeatHotMs, level > kHeatHotMs ? "low-power" : "boost");
    return level > kHeatHotMs;
}

double power_heat_ms() {  // diagnostics: the policy's current input on the current device
    Heat& h = heat_here();
    const auto now = std::chrono::steady_clock::now();
    std::lock_guard<std::mutex> lk(h.mu);
    return decayed(h, now);
}

int effective_xt_variant() {
    const long v = g_opt_xt_variant.load();
    if (v != 0) return int(v);          // explicit measurement override
    return low_power_now() ? 2 : 0;
}

static double est_ms_for(const SwecApplyParams& p, int k, int r) {
    return double(p.nvec) * 16.0 * double(k + r) / 3.0e12 * 1e3;   // algorithmic bytes at ~3.0 TB/s (H100 SXM HBM3)
}

int encode_ctas_per_sm() {
    const long c = g_opt_ctas_per_sm.load();
    if (c > 0 && c <= 64) return int(c);
    const long t = g_opt_enc_threads.load(), u = g_opt_enc_unroll.load();
    // ≈768 resident threads per SM with one column slice per thread, ≈512 with two: the rule an earlier GPU generation's
    // sweep chose; on an H100 SXM every swept shape lies within 4 % of the others (scripts/tune_encode.py)
    const long tt = t == 128 || t == 512 ? t : 256;
    return int(std::max(1l, (u > 1 ? 512 : 768) / tt));
}

template <int THREADS, int UNROLL>
static cudaError_t launch_rs10x4_shape(const SwecApplyParams& p, bool blocked, int ctas_per_sm, cudaStream_t s) {
    const unsigned grid = grid_for((p.nvec + UNROLL - 1) / UNROLL, THREADS, ctas_per_sm);
    const bool lp = low_power_now();
    note_kernel_work(est_ms_for(p, 10, 4));
    if (blocked && lp) rs10x4_encode<THREADS, UNROLL, true, true><<<grid, THREADS, 0, s>>>(p);
    else if (blocked) rs10x4_encode<THREADS, UNROLL, true, false><<<grid, THREADS, 0, s>>>(p);
    else if (lp) rs10x4_encode<THREADS, UNROLL, false, true><<<grid, THREADS, 0, s>>>(p);
    else rs10x4_encode<THREADS, UNROLL, false, false><<<grid, THREADS, 0, s>>>(p);
    return launched();
}

cudaError_t launch_rs10x4_encode(const SwecApplyParams& p, bool blocked, cudaStream_t s) {
    if (p.nvec == 0) return cudaSuccess;
    const long threads = g_opt_enc_threads.load(), unroll = g_opt_enc_unroll.load();
    const int c = encode_ctas_per_sm();
    if (threads == 128 && unroll == 1) return launch_rs10x4_shape<128, 1>(p, blocked, c, s);
    if (threads == 128 && unroll == 2) return launch_rs10x4_shape<128, 2>(p, blocked, c, s);
    if (threads == 512 && unroll == 1) return launch_rs10x4_shape<512, 1>(p, blocked, c, s);
    if (threads == 512 && unroll == 2) return launch_rs10x4_shape<512, 2>(p, blocked, c, s);
    if (unroll == 2) return launch_rs10x4_shape<256, 2>(p, blocked, c, s);
    return launch_rs10x4_shape<256, 1>(p, blocked, c, s);
}

cudaError_t launch_table_apply(const SwecApplyParams& p, const u32* replicated_tables, int K, int r, cudaStream_t s) {
    if (p.nvec == 0) return cudaSuccess;
    const size_t smem = size_t(K) * 4096;
    const int per_sm = smem <= 56 * 1024 ? 4 : (smem <= 113 * 1024 ? 2 : 1);
    const unsigned grid = grid_for(p.nvec, 256, per_sm);
    cudaError_t e;
    if (K == 10) {
        e = cudaFuncSetAttribute(swec_table_kernel<10>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess) return e;
        swec_table_kernel<10><<<grid, 256, smem, s>>>(p, replicated_tables, K, r);
    } else {
        e = cudaFuncSetAttribute(swec_table_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess) return e;
        swec_table_kernel<0><<<grid, 256, smem, s>>>(p, replicated_tables, K, r);
    }
    return launched();
}

cudaError_t launch_bytes_apply(const SwecApplyParams& p, const u32* compact_tables, int K, int r, u64 nbytes,
                               cudaStream_t s) {
    if (nbytes == 0) return cudaSuccess;
    swec_bytes_kernel<<<grid_for(nbytes, 256, 8), 256, 0, s>>>(p, compact_tables, K, r, nbytes);
    return launched();
}

cudaError_t launch_synth(void* dst, u64 byte_offset, u64 nbytes, u64 seed, cudaStream_t s) {
    if (nbytes == 0) return cudaSuccess;
    swec_synth_kernel<<<grid_for(nbytes / 8, 256, 8), 256, 0, s>>>(static_cast<u64*>(dst), byte_offset / 8, nbytes / 8, seed);
    return launched();
}

cudaError_t launch_digest(const void* src, u64 nbytes, u64* out_dev, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(out_dev, 0, 8, s);
    if (e != cudaSuccess || nbytes == 0) return e;
    swec_digest_kernel<<<grid_for((nbytes + 7) / 8, 256, 8), 256, 0, s>>>(static_cast<const u8*>(src), nbytes, out_dev);
    return launched();
}

cudaError_t launch_compare(const void* a, const void* b, u64 nbytes, unsigned long long* out_dev, cudaStream_t s) {
    if (nbytes == 0) return cudaSuccess;
    swec_compare_kernel<<<grid_for((nbytes + 15) / 16, 256, 8), 256, 0, s>>>(static_cast<const u8*>(a), static_cast<const u8*>(b), nbytes, out_dev);
    return launched();
}

}  // namespace swec
