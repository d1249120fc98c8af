// seaweedfs_b200/csrc/sketch.cu — page sketches of shards, and damage located from the sketches of a whole set.
//
//   swec_page_sketch_kernel   one warp per 4 KiB page, grid-stride.  Bit-sliced: a lane keeps eight words T_b, T_b the
//                             XOR of the weight words w(x) of its columns whose byte has bit b set, so each column costs
//                             one splitmix64 and eight masked XORs.  The lane's share of the page is then
//                             ⊕_b 2^b ⊗ T_b (Horner over b with a multiply-by-2 on all 8 bytes at once), and the warp
//                             XORs its 32 shares with shuffles.  A whole page of an aligned shard is read as 8 coalesced
//                             16-byte loads per lane; the partial last page and unaligned shards go byte by byte.
//   swec_sketch_pages_kernel  the page decode of both sketch calls, over the errors-and-erasures plan of the present
//                             shards (damage.h): one thread per page, the 8 bytes of its sketch syndromes decoded as 8
//                             columns by the locate kernels' decoder (locate_decode.cuh), their blame merged per page,
//                             and the located errors of information shards taken out of the lost shards' sketches.
//   swec_sketch_attribute_kernel  the needles that flagged pages hit: one thread per (flagged page, data shard), which
//                             cuts the page's columns of that shard into runs of consecutive .dat offsets (one run
//                             when both block sizes are multiples of 4096), binary-searches each run's first candidate
//                             record and walks the offset-sorted records forward, one atomic per (record, run).  Work
//                             grows with the records a page overlaps, not with its 4096 bytes: a whole 3 GiB shard
//                             flagged is 786,432 threads, not 3.2 G byte lookups.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "damage.h"
#include "device_common.cuh"
#include "engine.h"
#include "locate_decode.cuh"
#include "needle_damage.h"
#include "sketch.h"

namespace swec {

namespace {

constexpr u64 kPage = 4096;
constexpr u64 kGolden = 0x9E3779B97F4A7C15ull;  // splitmix64's increment: w(x) = mix(seed + (x+1)·kGolden)

__device__ __forceinline__ u64 mix(u64 z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// column with byte c and weight word w into the slices
__device__ __forceinline__ void take(u64 (&t)[8], u64 w, u32 c) {
#pragma unroll
    for (int b = 0; b < 8; b++) t[b] ^= w & (0ull - u64((c >> b) & 1u));
}

// 2 ⊗ every byte of a (GF(2^8)/0x11D)
__device__ __forceinline__ u64 xtime8(u64 a) {
    return ((a & 0x7f7f7f7f7f7f7f7full) << 1) ^ (((a >> 7) & 0x0101010101010101ull) * 0x1d);
}

__global__ void __launch_bounds__(256) swec_page_sketch_kernel(const u8* __restrict__ src, u64 n, u64 first_column,
                                                               u64 seed, u64* __restrict__ out) {
    const u64 pages = (n + kPage - 1) / kPage;
    const u32 lane = threadIdx.x & 31;
    const u64 warps = (u64)gridDim.x * (blockDim.x >> 5);
    const bool vec = (reinterpret_cast<unsigned long long>(src) & 15) == 0;
    for (u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < pages; g += warps) {
        const u64 p0 = g * kPage;
        const u64 len = min(kPage, n - p0);
        const u64 z0 = seed + (first_column + p0 + 1) * kGolden;  // before mix: the weight of the page's first column
        u64 t[8];
#pragma unroll
        for (int b = 0; b < 8; b++) t[b] = 0;
        if (vec && len == kPage) {
            uint4 d[8];
#pragma unroll
            for (int j = 0; j < 8; j++) d[j] = swec_ldg_stream(src + p0 + (u64(lane + 32 * j) << 4));
#pragma unroll
            for (int j = 0; j < 8; j++) {
                u64 z = z0 + u64((lane + 32 * j) << 4) * kGolden;
                const u32 w[4] = {d[j].x, d[j].y, d[j].z, d[j].w};
#pragma unroll
                for (int c = 0; c < 16; c++, z += kGolden) take(t, mix(z), w[c >> 2] >> (8 * (c & 3)));
            }
        } else {
            for (u32 x = lane; x < len; x += 32) take(t, mix(z0 + u64(x) * kGolden), src[p0 + x]);
        }
        u64 r = t[7];
#pragma unroll
        for (int b = 6; b >= 0; b--) r = xtime8(r) ^ t[b];
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, s);
        if (lane == 0) out[g] = r;
    }
}

struct SketchPageParams {
    const u64* comp[SWEC_MAX_SHARDS];    // check sketches recomputed from the information sketches
    const u64* stored[SWEC_MAX_SHARDS];  // check sketches as their holders sent them
    u64* rebuilt[SWEC_MAX_SHARDS];       // R·(information sketches) of every lost shard, corrected in place
    u8 ids[SWEC_MAX_SHARDS];             // shard id of every position: information 0..k-1, checks k..k+c-1
    u64 pages;
    int k, c, f, radius;                 // information, check and lost shards; the radius, at most c/2
    const u32* tables;                   // LocateTables of the check rows P', then log R (kLogRWords, f > 0)
    swec_sketch_page* flagged;           // one entry per flagged page, in no particular order
    unsigned long long* count;           // entries written
};

// R[r][j]·e, the image in lost shard r of error value e at information position j (0 for any other position)
__device__ __forceinline__ u8 carried(const LocateTables& t, const u8* logr, int r, u32 j, u8 e, int k) {
    if (j >= u32(k) || !e) return 0;
    const u8 lr = logr[r * 32 + int(j)];
    return lr == kLogZero ? 0 : t.exp[lr + t.log[e]];
}

// Page decode, one thread per page, grid-stride.  Byte l of the c sketch syndromes of page g is the syndrome of sketch
// column (g, l): each non-zero column is decoded as the locate kernel decodes a byte column, and the page is blamed on
// the union of its columns' blame, or uncorrectable when a column is or the union exceeds the radius.  Radius 0
// decodes nothing.  The positions and error values of the 8 columns are kept a byte each in four words, and only a
// page decoded within the radius XORs the images of its information errors into byte l of every lost shard's sketch
// word; an uncorrectable page keeps R·(information sketches as found).  Clean pages cost the loads.
__global__ void __launch_bounds__(256) swec_sketch_pages_kernel(const __grid_constant__ SketchPageParams p) {
    __shared__ __align__(16) u32 words[kTableWords + kLogRWords];
    const int n_words = kTableWords + (p.f > 0 ? kLogRWords : 0);
    for (int i = threadIdx.x; i < n_words; i += blockDim.x) words[i] = p.tables[i];
    __syncthreads();
    const LocateTables& t = *reinterpret_cast<const LocateTables*>(words);
    const u8* logr = reinterpret_cast<const u8*>(words + kTableWords);
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < p.pages; g += stride) {
        u64 any = 0;
        for (int i = 0; i < p.c; i++) any |= p.comp[i][g] ^ p.stored[i][g];
        if (!any) continue;
        u32 mask = 0;                      // blamed positions
        bool bad = false;
        u64 pa = ~0ull, pb = ~0ull;        // byte l: the positions column l is blamed on, 0xff for none
        u64 va = 0, vb = 0;                // byte l: their error values
        for (int l = 0; l < 8 && !bad; l++) {
            u8 s[SWEC_MAX_SHARDS];
            u8 nz = 0;
            for (int i = 0; i < p.c; i++) {
                s[i] = u8((p.comp[i][g] ^ p.stored[i][g]) >> (8 * l));
                nz |= s[i];
            }
            if (!nz) continue;
            int a = -1, b = -1;
            u8 ea = 0, eb = 0;
            const int found = p.radius == 0 ? 0 : decode_column<true>(t, s, p.k, p.c, p.radius, &a, &b, &ea, &eb);
            bad = !found;
            if (found >= 1) {
                mask |= 1u << a;
                pa ^= u64(0xff ^ a) << (8 * l);
                va |= u64(ea) << (8 * l);
            }
            if (found == 2) {
                mask |= 1u << b;
                pb ^= u64(0xff ^ b) << (8 * l);
                vb |= u64(eb) << (8 * l);
            }
        }
        bad = bad || __popc(mask) > p.radius;
        u32 blamed = 0;  // the shard ids of the blamed positions
        for (u32 x = bad ? 0u : mask; x; x &= x - 1) blamed |= 1u << p.ids[__ffs(x) - 1];
        const unsigned long long at = atomicAdd(p.count, 1ull);
        p.flagged[at].page = int64_t(g);
        p.flagged[at].blamed_mask = blamed;
        p.flagged[at].uncorrectable = bad ? 1 : 0;
        if (bad) continue;
        for (int r = 0; r < p.f; r++) {
            u64 fix = 0;
            for (int l = 0; l < 8; l++) {
                const int sh = 8 * l;
                const u8 x = carried(t, logr, r, u32(pa >> sh) & 0xff, u8(va >> sh), p.k) ^
                             carried(t, logr, r, u32(pb >> sh) & 0xff, u8(vb >> sh), p.k);
                fix |= u64(x) << sh;
            }
            p.rebuilt[r][g] ^= fix;
        }
    }
}

// Both sketch calls: sketches[id] are the host sketches of the present shards (n_pages words each), decoded over
// `plan` at plan.radius(radius).  One apply of plan.fused to the uploaded information sketches gives the check sketches
// and R·(information sketches) of every lost shard; the page decode (c >= 1) compares the check sketches with the
// stored ones and corrects the lost shards' sketches.  The flagged pages come back in ascending page order, and the
// sketch of lost shard id into out[id] where out and out[id] are non-NULL.  Synchronous on the encoder's stream.
int sketch_pages(swec_encoder* e, const CheckedPlan& plan, const uint64_t* const* sketches, int64_t n_pages, int radius,
                 uint64_t* const* out, std::vector<swec_sketch_page>* flagged) {
    const int k = e->k, c = plan.c(), nout = int(plan.outs.size()), f = int(plan.rebuilt_rows.size());
    flagged->clear();
    if (n_pages == 0) return SWEC_OK;
    cudaStream_t s = e->stream;
    const size_t bytes = size_t(n_pages) * 8, pitch = (bytes + 15) & ~size_t(15);  // 16-byte rows: the vector path
    // the k information and c check sketches as uploaded, then the nout rows the apply computes
    StreamScratch buf(s);
    SWEC_CUDA(buf.alloc(size_t(k + c + nout) * pitch));
    auto row = [&](int i) { return buf.as<uint8_t>() + size_t(i) * pitch; };
    uint8_t* at[SWEC_MAX_SHARDS];
    uint8_t* comp[SWEC_MAX_SHARDS];
    for (int i = 0; i < k + c; i++) {
        at[i] = row(i);
        SWEC_CUDA(cudaMemcpyAsync(at[i], sketches[i < k ? plan.info[size_t(i)] : plan.check(i - k)], bytes,
                                  cudaMemcpyHostToDevice, s));
    }
    for (int o = 0; o < nout; o++) comp[o] = row(k + c + o);
    // sketches are linear: the plan's rows applied to the information sketches give every other shard's clean sketch
    if (int rc = e->apply(plan.fused, at, comp, bytes, Layout{}, s)) return rc;
    if (c > 0) {
        std::vector<u8> host(sizeof(LocateTables) + kLogRBytes);
        locate_tables(plan.checks(), reinterpret_cast<LocateTables*>(host.data()));
        plan.rebuilt_logs(host.data() + sizeof(LocateTables));
        DeviceBuffer tables;
        SWEC_CUDA(tables.upload(host.data(), host.size(), s));
        StreamScratch res(s);
        SWEC_CUDA(res.alloc(sizeof(unsigned long long) + size_t(n_pages) * sizeof(swec_sketch_page)));
        SketchPageParams p;
        memset(&p, 0, sizeof p);
        for (int i = 0; i < c; i++) {
            p.comp[i] = reinterpret_cast<const u64*>(comp[plan.check_rows[size_t(i)]]);
            p.stored[i] = reinterpret_cast<const u64*>(at[k + i]);
            p.ids[k + i] = u8(plan.check(i));
        }
        for (int j = 0; j < k; j++) p.ids[j] = u8(plan.info[size_t(j)]);
        for (int r = 0; r < f; r++) p.rebuilt[r] = reinterpret_cast<u64*>(comp[plan.rebuilt_rows[size_t(r)]]);
        p.pages = u64(n_pages);
        p.k = k;
        p.c = c;
        p.f = f;
        p.radius = plan.radius(radius);
        p.tables = tables.as<u32>();
        p.count = res.as<unsigned long long>();
        p.flagged = reinterpret_cast<swec_sketch_page*>(p.count + 1);
        SWEC_CUDA(cudaMemsetAsync(p.count, 0, sizeof *p.count, s));
        static const int per_sm = [] {
            int n = 0;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, swec_sketch_pages_kernel, 256, 0) != cudaSuccess) {
                cudaGetLastError();
                n = 4;
            }
            return std::max(1, n);
        }();
        swec_sketch_pages_kernel<<<grid_for(u64(n_pages), 256, per_sm), 256, 0, s>>>(p);
        SWEC_CUDA(launched());
        unsigned long long n = 0;
        SWEC_CUDA(cudaMemcpyAsync(&n, p.count, sizeof n, cudaMemcpyDeviceToHost, s));
        SWEC_CUDA(cudaStreamSynchronize(s));
        flagged->resize(size_t(n));
        if (n)
            SWEC_CUDA(cudaMemcpyAsync(flagged->data(), p.flagged, size_t(n) * sizeof(swec_sketch_page),
                                      cudaMemcpyDeviceToHost, s));
    }
    for (int r = 0; r < f && out; r++)
        if (uint64_t* dst = out[plan.rebuilt(r)])
            SWEC_CUDA(cudaMemcpyAsync(dst, comp[plan.rebuilt_rows[size_t(r)]], bytes, cudaMemcpyDeviceToHost, s));
    SWEC_CUDA(cudaStreamSynchronize(s));
    std::sort(flagged->begin(), flagged->end(),
              [](const swec_sketch_page& a, const swec_sketch_page& b) { return a.page < b.page; });
    return SWEC_OK;
}

// The tail of both sketch calls, after their argument rules: the decode over `plan`, then the caller's outputs.
int locate_sketches(swec_encoder* e, const CheckedPlan& plan, const uint64_t* const* sketches, int64_t shard_len,
                    int radius, swec_sketch_page* pages, int64_t pages_cap, int64_t* n_flagged, uint64_t* shard_pages,
                    uint64_t* const* rebuilt, int* ok) {
    std::lock_guard<std::mutex> lock(e->mu);
    if (int rc = e->ensure_device()) return rc;
    const int64_t n_pages = (shard_len + int64_t(kPage) - 1) / int64_t(kPage);
    std::vector<swec_sketch_page> flagged;
    if (int rc = sketch_pages(e, plan, sketches, n_pages, radius, rebuilt, &flagged)) return rc;
    if (shard_pages) memset(shard_pages, 0, SWEC_MAX_SHARDS * sizeof *shard_pages);
    for (size_t i = 0; i < flagged.size(); i++) {
        if (int64_t(i) < pages_cap) pages[i] = flagged[i];
        for (uint32_t b = flagged[i].blamed_mask; b && shard_pages; b &= b - 1) shard_pages[__builtin_ctz(b)]++;
    }
    *n_flagged = int64_t(flagged.size());
    *ok = plan.c() >= 1 && flagged.empty() ? 1 : 0;
    return SWEC_OK;
}

struct SketchAttributeParams {
    const swec_sketch_page* pages;  // flagged pages, ascending
    u64 n_pages;
    int64_t shard_len;
    StripeMap map;
    RecordTally t;
};

// One thread per (flagged page, data shard i), grid-stride.  A blamed page counts the columns of the data shards in its
// mask as damaged, an uncorrectable one the columns of all k data shards as uncorrectable; parity blame is never
// attributed.  Each block run of the page goes to its records by the ownership rule (RecordTally::owned), and the
// bytes no record owns, padding included, to the unowned counter of the kind, once per thread.
__global__ void __launch_bounds__(256) swec_sketch_attribute_kernel(const __grid_constant__ SketchAttributeParams p) {
    const u64 k = u64(p.map.k), total = p.n_pages * k;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += stride) {
        const u64 j = w / k;
        const int i = int(w - j * k);
        const swec_sketch_page pg = p.pages[j];
        const int kind = pg.uncorrectable ? 1 : 0;
        if (!kind && !((pg.blamed_mask >> i) & 1u)) continue;
        const int64_t lo = pg.page * int64_t(kPage), hi = min(lo + int64_t(kPage), p.shard_len);
        unsigned long long lost = 0;
        for (int64_t x = lo; x < hi;) {
            const int64_t stop = min(hi, p.map.block_end(x));
            const int64_t d0 = p.map.dat_offset(i, x);  // -1: the whole run is padding
            const int64_t len = stop - x;
            x = stop;
            if (d0 < 0) {
                lost += u64(len);
                continue;
            }
            const int64_t d1 = min(d0 + len, p.map.dat_end);
            int64_t got = 0;
            for (int q = max(p.t.candidate(d0), 0); q < p.t.n && p.t.off[q] < d1; q++) {
                const int64_t o = p.t.owned(q, d0, d1);
                if (!o) continue;
                atomicAdd((kind ? p.t.uncorrectable : p.t.damaged) + q, (unsigned long long)o);
                atomicOr(p.t.mask + q, 1u << i);
                got += o;
            }
            lost += u64(len - got);
        }
        if (lost) atomicAdd(p.t.unowned + kind, lost);
    }
}

}  // namespace

int check_sketch_pages(int k, int m, int64_t shard_len, const swec_sketch_page* pages, int64_t n_pages) {
    const int64_t limit = (shard_len + int64_t(kPage) - 1) / int64_t(kPage);
    const uint64_t shards = (uint64_t(1) << (k + m)) - 1;
    for (int64_t j = 0; j < n_pages; j++) {
        const swec_sketch_page& pg = pages[j];
        const std::string at = "pages[" + std::to_string(j) + "]";
        if (pg.page < 0 || pg.page >= limit || (j > 0 && pg.page <= pages[j - 1].page))
            return fail(SWEC_ERR_INVALID_ARG, at + ": pages must be strictly ascending and below ceil(shard_len/4096)");
        if (pg.uncorrectable != 0 && pg.uncorrectable != 1)
            return fail(SWEC_ERR_INVALID_ARG, at + ": uncorrectable must be 0 or 1");
        if (pg.uncorrectable ? pg.blamed_mask != 0 : (pg.blamed_mask == 0 || (pg.blamed_mask & ~shards)))
            return fail(SWEC_ERR_INVALID_ARG, at + ": an uncorrectable page has mask 0, a blamed page a non-zero mask "
                                                   "of the k+m shards");
    }
    return SWEC_OK;
}

int sketch_needle_damage(int device, const StripeMap& map, int64_t shard_len, const swec_sketch_page* pages,
                         int64_t n_pages, swec_needle_damage* recs, int n, int version, uint64_t unowned[2]) {
    SWEC_CUDA(cudaSetDevice(device));
    cudaStream_t s = cudaStreamPerThread;
    NeedleDamage nd;
    if (int rc = nd.init(map.k, 0, map, recs, n, version, 0, 0, s)) return rc;
    DeviceBuffer flagged;
    SWEC_CUDA(flagged.upload(pages, size_t(n_pages), s));
    SketchAttributeParams p;
    memset(&p, 0, sizeof p);
    p.pages = flagged.as<swec_sketch_page>();
    p.n_pages = u64(n_pages);
    p.shard_len = shard_len;
    p.map = map;
    p.t = nd.tally();
    static const int per_sm = [] {
        int c = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, swec_sketch_attribute_kernel, 256, 0) != cudaSuccess) {
            cudaGetLastError();
            c = 4;
        }
        return std::max(1, c);
    }();
    swec_sketch_attribute_kernel<<<grid_for(u64(n_pages) * u64(map.k), 256, per_sm), 256, 0, s>>>(p);
    SWEC_CUDA(launched());
    SWEC_CUDA(cudaStreamSynchronize(s));
    return nd.collect(recs, unowned);
}

cudaError_t launch_page_sketch(const void* shard, u64 n, u64 first_column, u64 seed, u64* sketches, cudaStream_t s) {
    if (n == 0) return cudaSuccess;
    static const int per_sm = [] {  // resident CTAs per SM, the same on every device of this architecture
        int c = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, swec_page_sketch_kernel, 256, 0) != cudaSuccess) {
            cudaGetLastError();
            c = 4;
        }
        return std::max(1, c);
    }();
    const u64 pages = (n + kPage - 1) / kPage;
    swec_page_sketch_kernel<<<grid_for(pages, 8, per_sm), 256, 0, s>>>(static_cast<const u8*>(shard), n, first_column,
                                                                       seed, sketches);
    return launched();
}

}  // namespace swec

using namespace swec;

extern "C" {

int swec_page_sketch_device(int device, const void* shard, size_t len, uint64_t first_column, uint64_t seed,
                            uint64_t* sketches, void* stream) {
    if (len > 0 && (!shard || !sketches)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    if (first_column % kPage) return fail(SWEC_ERR_INVALID_ARG, "first_column must be a multiple of 4096");
    if (reinterpret_cast<uintptr_t>(sketches) & 7) return fail(SWEC_ERR_INVALID_ARG, "sketches must be 8-byte aligned");
    if (device < 0) return fail(SWEC_ERR_NO_DEVICE, "device < 0; no CPU fallback exists");
    if (len == 0) return SWEC_OK;
    SWEC_CUDA(cudaSetDevice(device));
    SWEC_CUDA(launch_page_sketch(shard, len, first_column, seed, reinterpret_cast<u64*>(sketches),
                                 static_cast<cudaStream_t>(stream)));
    return SWEC_OK;
}

int swec_locate_sketch_damage(swec_encoder* e, const uint64_t* const* sketches, int64_t shard_len, int radius,
                              swec_sketch_page* pages, int64_t pages_cap, int64_t* n_flagged, uint64_t* shard_pages,
                              int* ok) {
    if (!e || !sketches || !n_flagged || !ok) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    if (shard_len < 0) return fail(SWEC_ERR_INVALID_ARG, "shard_len must be >= 0");
    if (pages_cap < 0 || (pages_cap > 0 && !pages))
        return fail(SWEC_ERR_INVALID_ARG, "pages_cap must be >= 0, and pages non-NULL when it is > 0");
    if (int rc = check_radius(radius, 0, e->m)) return rc;
    for (int i = 0; i < e->k + e->m; i++)
        if (!sketches[i])
            return fail(SWEC_ERR_TOO_FEW_SHARDS, "no sketch of shard " + std::to_string(i) + ": rebuild it first");
    return locate_sketches(e, CheckedPlan::all_present(e->gen, e->k), sketches, shard_len, radius, pages, pages_cap,
                           n_flagged, shard_pages, nullptr, ok);
}

int swec_locate_sketch_damage_checked(swec_encoder* e, const uint64_t* const* sketches, int64_t shard_len, int radius,
                                      swec_sketch_page* pages, int64_t pages_cap, int64_t* n_flagged,
                                      uint64_t* shard_pages, uint64_t* const* rebuilt_sketches, int* ok) {
    if (!e || !sketches || !n_flagged || !ok) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    if (shard_len < 0) return fail(SWEC_ERR_INVALID_ARG, "shard_len must be >= 0");
    if (pages_cap < 0 || (pages_cap > 0 && !pages))
        return fail(SWEC_ERR_INVALID_ARG, "pages_cap must be >= 0, and pages non-NULL when it is > 0");
    if (int rc = check_radius(radius, 0)) return rc;
    std::vector<uint8_t> present(size_t(e->k + e->m));
    for (size_t i = 0; i < present.size(); i++) present[i] = sketches[i] != nullptr;
    CheckedPlan plan;
    if (!plan.build(e->gen, e->k, present.data(), false))
        return fail(SWEC_ERR_TOO_FEW_SHARDS, "fewer than data_shards sketches present");
    return locate_sketches(e, plan, sketches, shard_len, radius, pages, pages_cap, n_flagged, shard_pages,
                           rebuilt_sketches, ok);
}

int swec_sketch_needle_damage(int device, int k, int m, int64_t shard_len, int64_t dat_size, int64_t large,
                              int64_t small, const swec_sketch_page* pages, int64_t n_pages, swec_needle_damage* records,
                              int n_records, uint64_t unowned[2]) {
    if (k <= 0 || m <= 0 || k + m > SWEC_MAX_SHARDS)
        return fail(SWEC_ERR_INVALID_ARG, "need data_shards > 0, parity_shards > 0, total <= 32");
    if (dat_size < 0 || large <= 0 || small <= 0) return fail(SWEC_ERR_INVALID_ARG, "bad geometry");
    if (shard_len != swec_expected_shard_size(dat_size, k, large, small))
        return fail(SWEC_ERR_INVALID_ARG, "shard_len " + std::to_string(shard_len) + " is not the shard size " +
                                              std::to_string(swec_expected_shard_size(dat_size, k, large, small)) +
                                              " of the geometry");
    if (n_pages < 0 || (n_pages > 0 && !pages))
        return fail(SWEC_ERR_INVALID_ARG, "n_pages must be >= 0, and pages non-NULL when it is > 0");
    int rc = check_needle_damage_args(0, nullptr, unowned, n_records, records);
    if (rc || (rc = check_sketch_pages(k, m, shard_len, pages, n_pages))) return rc;
    if (n_pages == 0) {
        for (int j = 0; j < n_records; j++) {
            records[j].shard_mask = 0;
            records[j].damaged_bytes = records[j].uncorrectable_bytes = 0;
        }
        unowned[0] = unowned[1] = 0;
        return SWEC_OK;
    }
    if (device < 0) return fail(SWEC_ERR_NO_DEVICE, "device < 0; no CPU fallback exists");
    return sketch_needle_damage(device, StripeMap::encode(dat_size, k, large, small), shard_len, pages, n_pages, records,
                                n_records, 3, unowned);
}

}  // extern "C"
