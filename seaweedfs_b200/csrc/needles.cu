// seaweedfs_b200/csrc/needles.cu — Needle.ReadBytes (weed/storage/needle/needle_read.go:59-190) on records resident
// in HBM: the size check, the layout walk of needle_format.h and the CRC32-C of Data (needle_read_tail.go:11-34,
// crc.go:12-22).  Four launches per batch, none of which follows the record size mix:
//   needle_parse_kernel   one thread per record: bounds, header Size, body layout, stored checksum, Data chunk count
//   needle_scan_kernel    one CTA: exclusive prefix sum of the chunk counts (where each record's chunks start)
//   needle_crc_kernel     one lane per 16 KiB chunk of Data, wherever it lies: raw CRC with slicing-by-4 tables,
//                         lane-replicated in shared memory (one TMA bulk copy per CTA, conflict-free for any data),
//                         shifted to the end of its record and XOR-ed into the record: crc(A‖B) = crc(A)·x^(8|B|) ⊕ crc(B)
//   needle_final_kernel   one thread per record: init/final XOR of the Castagnoli CRC, compare, legacy form
#include <cuda_runtime.h>

#include <cstdint>
#include <mutex>

#include "engine.h"
#include "needle_format.h"
#include "needles.h"
#include "tma_fetch.cuh"

namespace swec {

namespace {

constexpr u32 kCastagnoli = 0x82F63B78u;  // reflected polynomial
constexpr u32 kChunk = 16384;              // bytes of Data one lane checksums before joining
constexpr int kCrcThreads = 1024;
constexpr u32 kTableBytes = 4u * 256u * 32u * 4u;  // slicing-by-4, one copy per lane: 128 KiB
constexpr int kPowers = 40;                        // x^(8·2^j) mod P for j < 40: shifts of up to 2^40 bytes

// a·b mod P in the reflected representation (bit 31 = x^0), a != 0
__device__ __forceinline__ u32 multmodp(u32 a, u32 b) {
    u32 m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = (b & 1) ? (b >> 1) ^ kCastagnoli : b >> 1;
    }
    return p;
}

// x^(8n) mod P: the factor that moves a CRC register over n more bytes
__device__ __forceinline__ u32 xpow8(const u32* __restrict__ powers, u64 n) {
    u32 p = 1u << 31;
    for (int j = 0; n; j++, n >>= 1)
        if (n & 1) p = multmodp(__ldg(powers + j), p);
    return p;
}

// T_k[i] word k*256+i of lane l at word ((k*256+i) << 5) | l: lane l always reads bank l
__global__ void needle_tables_kernel(u32* __restrict__ replicated, u32* __restrict__ powers) {
    __shared__ u32 t[4][256];
    const int i = threadIdx.x;
    u32 c = u32(i);
    for (int b = 0; b < 8; b++) c = (c & 1) ? (c >> 1) ^ kCastagnoli : c >> 1;
    t[0][i] = c;
    __syncthreads();
    for (int k = 1; k < 4; k++) {
        t[k][i] = (t[k - 1][i] >> 8) ^ t[0][t[k - 1][i] & 0xffu];
        __syncthreads();
    }
    for (int k = 0; k < 4; k++)
        for (int l = 0; l < 32; l++) replicated[((k * 256 + i) << 5) | l] = t[k][i];
    if (i == 0) {
        u32 p = 1u << 30;  // x^1
        p = multmodp(p, p);
        p = multmodp(p, p);  // x^4
        for (int j = 0; j < kPowers; j++) {
            p = multmodp(p, p);
            powers[j] = p;
        }
    }
}

__global__ void needle_parse_kernel(const u8* __restrict__ dat, int64_t dat_size, int version,
                                    swec_needle_check* __restrict__ checks, int n, u64* __restrict__ first_chunk) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0) first_chunk[0] = 0;
    if (r >= n) return;
    swec_needle_check& c = checks[r];
    c.range_index = 0;
    c.data_size = 0;
    c.crc_got = 0;
    c.crc_want = 0;
    c.legacy_crc = 0;
    u64 chunks = 0;
    const int64_t off = c.offset;
    const int64_t need = c.size < 0 ? kNeedleHeaderSize : needle_actual_size(c.size, version);  // < 0: a size mismatch
    if (off < 0 || off > dat_size || need > dat_size - off) {
        c.status = SWEC_NEEDLE_OUTSIDE_IMAGE;
    } else {
        const RecordLayout l = record_layout(dat + off, c.size, version);
        c.status = l.status;
        c.range_index = l.range_index;
        c.data_size = l.data_size;
        c.crc_want = l.crc_want;
        if (l.status == SWEC_NEEDLE_OK) chunks = (u64(l.data_size) + kChunk - 1) / kChunk;
    }
    first_chunk[r + 1] = chunks;
}

// a[1..n] ← inclusive prefix sums, in tiles of 1024
__global__ void __launch_bounds__(1024) needle_scan_kernel(u64* __restrict__ a, int n) {
    __shared__ u64 warp_sums[32];
    __shared__ u64 carry;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + threadIdx.x;
        u64 v = i < n ? a[i + 1] : 0;
        for (int d = 1; d < 32; d <<= 1) {
            const u64 t = __shfl_up_sync(0xffffffffu, v, d);
            if (lane >= d) v += t;
        }
        if (lane == 31) warp_sums[w] = v;
        __syncthreads();
        if (w == 0) {
            u64 s = warp_sums[lane];
            for (int d = 1; d < 32; d <<= 1) {
                const u64 t = __shfl_up_sync(0xffffffffu, s, d);
                if (lane >= d) s += t;
            }
            warp_sums[lane] = s;
        }
        __syncthreads();
        v += carry + (w ? warp_sums[w - 1] : 0);
        if (i < n) a[i + 1] = v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = v;
        __syncthreads();
    }
}

// table k, index i of this lane's copy (tl = the table base + lane*4)
__device__ __forceinline__ u32 tab(const char* tl, u32 k, u32 i) {
    return *reinterpret_cast<const u32*>(tl + (((k << 8) | i) << 7));
}
__device__ __forceinline__ u32 crc_byte(const char* tl, u32 crc, u32 b) { return tab(tl, 0, (crc ^ b) & 0xffu) ^ (crc >> 8); }
__device__ __forceinline__ u32 crc_word(const char* tl, u32 crc, u32 w) {
    const u32 c = crc ^ w;
    return tab(tl, 3, c & 0xffu) ^ tab(tl, 2, (c >> 8) & 0xffu) ^ tab(tl, 1, (c >> 16) & 0xffu) ^ tab(tl, 0, c >> 24);
}

// raw CRC (register starts at 0, no final XOR) of [p, p+len): unaligned head by bytes, then 64 bytes per step in four
// 16-byte loads, then words and bytes
__device__ __forceinline__ u32 crc_raw(const char* tl, const u8* p, u32 len) {
    const u8* e = p + len;
    u32 crc = 0;
    while (p < e && (reinterpret_cast<uintptr_t>(p) & 15)) crc = crc_byte(tl, crc, *p++);
    while (e - p >= 64) {
        uint4 v[4];
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] = __ldg(reinterpret_cast<const uint4*>(p) + j);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            crc = crc_word(tl, crc, v[j].x);
            crc = crc_word(tl, crc, v[j].y);
            crc = crc_word(tl, crc, v[j].z);
            crc = crc_word(tl, crc, v[j].w);
        }
        p += 64;
    }
    while (e - p >= 4) {
        crc = crc_word(tl, crc, __ldg(reinterpret_cast<const u32*>(p)));
        p += 4;
    }
    while (p < e) crc = crc_byte(tl, crc, *p++);
    return crc;
}

__global__ void __launch_bounds__(kCrcThreads, 1)
    needle_crc_kernel(const u8* __restrict__ dat, int version, swec_needle_check* __restrict__ checks, int n,
                      const u64* __restrict__ first_chunk, const u32* __restrict__ tables, const u32* __restrict__ powers) {
    extern __shared__ __align__(128) u32 smem_tab[];
    __shared__ __align__(8) u64 mbar;
    tma_fetch(smem_tab, tables, kTableBytes, &mbar);
    const char* tl = reinterpret_cast<const char*>(smem_tab) + (threadIdx.x & 31u) * 4u;
    const int data_at = version == 1 ? kNeedleHeaderSize : kNeedleHeaderSize + kDataSizeSize;
    const u64 total = first_chunk[n];
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += stride) {
        int lo = 0, hi = n;  // first_chunk[lo] <= g < first_chunk[hi]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (first_chunk[mid] <= g) lo = mid;
            else hi = mid;
        }
        const u64 at = (g - first_chunk[lo]) * kChunk;
        const u32 len = checks[lo].data_size;
        const u32 clen = u32(min(u64(kChunk), u64(len) - at));
        u32 crc = crc_raw(tl, dat + checks[lo].offset + data_at + at, clen);
        const u64 after = u64(len) - at - clen;
        if (crc && after) crc = multmodp(xpow8(powers, after), crc);
        if (crc) atomicXor(&checks[lo].crc_got, crc);
    }
}

// Value() (crc.go:25-27): the form checksums were stored in before SeaweedFS 3.09
__device__ __forceinline__ u32 legacy_value(u32 c) { return ((c >> 15) | (c << 17)) + 0xa282ead8u; }

__global__ void needle_final_kernel(swec_needle_check* __restrict__ checks, int n, const u32* __restrict__ powers) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    swec_needle_check& c = checks[r];
    if (c.status != SWEC_NEEDLE_OK || c.data_size == 0) return;  // no Data: ReadBytes reads the checksum unchecked
    const u32 got = c.crc_got ^ multmodp(xpow8(powers, c.data_size), 0xffffffffu) ^ 0xffffffffu;
    c.crc_got = got;
    if (got != c.crc_want) {
        c.status = SWEC_NEEDLE_BAD_CRC;
        c.legacy_crc = legacy_value(got) == c.crc_want;
    }
}

struct Tables {
    u32* replicated = nullptr;
    u32* powers = nullptr;
};
std::mutex g_tables_mu;
Tables g_tables[64];  // per device, built on first use, kept for the life of the process

cudaError_t tables_for_current_device(Tables* out, cudaStream_t s) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    std::lock_guard<std::mutex> lk(g_tables_mu);
    Tables& t = g_tables[dev];
    if (!t.replicated) {
        u32* rep = nullptr;
        u32* pw = nullptr;
        e = cudaMalloc(reinterpret_cast<void**>(&rep), kTableBytes + kPowers * sizeof(u32));
        if (e != cudaSuccess) return e;
        pw = rep + kTableBytes / sizeof(u32);
        needle_tables_kernel<<<1, 256, 0, s>>>(rep, pw);
        e = launched();
        if (e == cudaSuccess) e = cudaFuncSetAttribute(needle_crc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kTableBytes));
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) {
            cudaFree(rep);
            return e;
        }
        t.replicated = rep;
        t.powers = pw;
    }
    *out = t;
    return cudaSuccess;
}

}  // namespace

size_t needle_check_scratch_bytes(int n) { return (size_t(n) + 1) * sizeof(u64); }

cudaError_t launch_needle_check(const void* dat, int64_t dat_size, int version, swec_needle_check* checks, int n,
                                void* scratch, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    Tables t;
    cudaError_t e = tables_for_current_device(&t, s);
    if (e != cudaSuccess) return e;
    const u8* d = static_cast<const u8*>(dat);
    u64* first_chunk = static_cast<u64*>(scratch);
    const unsigned per_record = unsigned((n + 255) / 256);
    needle_parse_kernel<<<per_record, 256, 0, s>>>(d, dat_size, version, checks, n, first_chunk);
    needle_scan_kernel<<<1, 1024, 0, s>>>(first_chunk, n);
    needle_crc_kernel<<<sm_count(), kCrcThreads, kTableBytes, s>>>(d, version, checks, n, first_chunk, t.replicated, t.powers);
    needle_final_kernel<<<per_record, 256, 0, s>>>(checks, n, t.powers);
    return launched(4);
}

}  // namespace swec

using namespace swec;

extern "C" int swec_check_needles_device(int device, const void* dat, int64_t dat_size, int needle_version,
                                         swec_needle_check* checks, int n, void* stream) {
    if (n < 0 || (n > 0 && (!checks || !dat)) || dat_size < 0) return fail(SWEC_ERR_INVALID_ARG, "NULL argument or negative size");
    if (needle_version < 1 || needle_version > 3) return fail(SWEC_ERR_INVALID_ARG, "needle version must be 1, 2 or 3");
    if (device < 0) return fail(SWEC_ERR_NO_DEVICE, "no CUDA device given: needle checks run on the GPU only");
    if (n == 0) return SWEC_OK;
    SWEC_CUDA(cudaSetDevice(device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const size_t table_bytes = size_t(n) * sizeof(swec_needle_check);
    StreamScratch buf(s);
    SWEC_CUDA(buf.alloc(table_bytes + needle_check_scratch_bytes(n)));
    auto* dev_checks = buf.as<swec_needle_check>();
    SWEC_CUDA(cudaMemcpyAsync(dev_checks, checks, table_bytes, cudaMemcpyHostToDevice, s));
    SWEC_CUDA(launch_needle_check(dat, dat_size, needle_version, dev_checks, n, buf.as<uint8_t>() + table_bytes, s));
    SWEC_CUDA(cudaMemcpyAsync(checks, dev_checks, table_bytes, cudaMemcpyDeviceToHost, s));
    SWEC_CUDA(cudaStreamSynchronize(s));
    return SWEC_OK;
}
