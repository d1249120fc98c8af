// seaweedfs_b200/csrc/needle_damage.cu — which needles the located damage hits (needle_damage.h), and the device call.
//
//   nd_attribute_kernel   grid-stride, one thread per byte column of a piece.  The column is uncorrectable when its
//                         residual syndrome (parity re-encoded from the corrected data XOR the corrected parity) is not
//                         zero: every column the correcting locate decoded within the radius is a codeword again.  A
//                         data byte is damaged when the correcting locate changed it: a blamed byte always changes,
//                         because its error value is not zero.  Each such byte of data shard i is mapped to its .dat
//                         offset (stripe_map.h), its owner among the live records is found by the ownership rule
//                         (RecordTally, needle_damage.h), and the owner's counters and shard mask, or the unowned
//                         counters, take it with atomics.
// The locate kernel itself (damage.cu) is not changed: pass 2 runs its correcting instantiation on a copy.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <numeric>

#include "damage.h"
#include "device_common.cuh"
#include "engine.h"
#include "needle_damage.h"
#include "needle_format.h"

namespace swec {

namespace {

struct AttributeParams {
    const u8* orig[SWEC_MAX_SHARDS];    // data shards as found
    const u8* fixed[SWEC_MAX_SHARDS];   // data shards after the correcting locate
    const u8* comp[SWEC_MAX_SHARDS];    // parity re-encoded from fixed
    const u8* stored[SWEC_MAX_SHARDS];  // parity after the correcting locate
    u64 n;
    int64_t base;
    int k, m;
    StripeMap map;
    RecordTally t;
};

__global__ void __launch_bounds__(256) nd_attribute_kernel(const __grid_constant__ AttributeParams p) {
    const u64 stride = u64(gridDim.x) * blockDim.x;
    for (u64 x = u64(blockIdx.x) * blockDim.x + threadIdx.x; x < p.n; x += stride) {
        u8 residual = 0;
        for (int q = 0; q < p.m; q++) residual |= p.comp[q][x] ^ p.stored[q][x];
        for (int i = 0; i < p.k; i++) {
            if (!residual && p.orig[i][x] == p.fixed[i][x]) continue;
            const int kind = residual ? 1 : 0;
            const int owner = p.t.owner(p.map.dat_offset(i, p.base + int64_t(x)));
            if (owner < 0) {
                atomicAdd(p.t.unowned + kind, 1ull);
                continue;
            }
            atomicAdd((kind ? p.t.uncorrectable : p.t.damaged) + owner, 1ull);
            atomicOr(p.t.mask + owner, 1u << i);
        }
    }
}

}  // namespace

int check_needle_damage_args(int needles_cap, const swec_needle_damage* needles, const uint64_t* unowned, int n_records,
                             const swec_needle_damage* records) {
    if (needles_cap < 0 || (needles_cap > 0 && !needles))
        return fail(SWEC_ERR_INVALID_ARG, "needles_cap must be >= 0, and needles non-NULL when it is > 0");
    if (!unowned) return fail(SWEC_ERR_INVALID_ARG, "unowned is NULL");
    if (n_records < 0 || (n_records > 0 && !records))
        return fail(SWEC_ERR_INVALID_ARG, "n_records must be >= 0, and records non-NULL when it is > 0");
    return SWEC_OK;
}

int NeedleDamage::init(int k, int m, const StripeMap& map, const swec_needle_damage* recs, int n, int version, int slots,
                       size_t piece, cudaStream_t s) {
    k_ = k;
    m_ = m;
    n_ = n;
    map_ = map;
    piece_ = piece;
    order_.resize(size_t(n));
    std::iota(order_.begin(), order_.end(), 0);
    std::stable_sort(order_.begin(), order_.end(), [&](int a, int b) { return recs[a].offset < recs[b].offset; });
    std::vector<int64_t> spans(size_t(2 * std::max(n, 1)), 0);
    for (int j = 0; j < n; j++) {
        const swec_needle_damage& r = recs[order_[size_t(j)]];
        spans[size_t(j)] = r.offset;
        spans[size_t(n + j)] = r.size < 0 ? r.offset : r.offset + needle_actual_size(r.size, version);
    }
    const size_t nc = size_t(2 * n + 2);
    SWEC_CUDA(counters_.alloc(nc * sizeof(unsigned long long)));
    SWEC_CUDA(masks_.alloc(size_t(std::max(n, 1)) * sizeof(unsigned)));
    if (slots > 0 && piece > 0) SWEC_CUDA(saved_.alloc(size_t(slots) * size_t(k) * piece));
    SWEC_CUDA(cudaMemsetAsync(counters_.as<void>(), 0, nc * sizeof(unsigned long long), s));
    SWEC_CUDA(cudaMemsetAsync(masks_.as<void>(), 0, size_t(std::max(n, 1)) * sizeof(unsigned), s));
    SWEC_CUDA(spans_.upload(spans.data(), spans.size(), s));  // synchronises s, after the clears
    return SWEC_OK;
}

int NeedleDamage::save(uint8_t* const* shards, size_t len, int slot, cudaStream_t s) {
    uint8_t* at = saved_.as<uint8_t>() + size_t(slot) * size_t(k_) * piece_;
    for (int i = 0; i < k_; i++)
        SWEC_CUDA(cudaMemcpyAsync(at + size_t(i) * piece_, shards[i], len, cudaMemcpyDeviceToDevice, s));
    return SWEC_OK;
}

int NeedleDamage::launch(const uint8_t* const* orig, uint8_t* const* fixed, uint8_t* const* comp, size_t len, int64_t base,
                         int slot, cudaStream_t s) {
    if (len == 0) return SWEC_OK;
    AttributeParams p;
    memset(&p, 0, sizeof p);
    for (int i = 0; i < k_; i++) {
        p.orig[i] = orig ? orig[i] : saved_.as<uint8_t>() + (size_t(slot) * size_t(k_) + size_t(i)) * piece_;
        p.fixed[i] = fixed[i];
    }
    for (int q = 0; q < m_; q++) {
        p.comp[q] = comp[q];
        p.stored[q] = fixed[k_ + q];
    }
    p.n = len;
    p.base = base;
    p.k = k_;
    p.m = m_;
    p.map = map_;
    p.t = tally();
    nd_attribute_kernel<<<grid_for(len, 256, 8), 256, 0, s>>>(p);
    SWEC_CUDA(launched());
    return SWEC_OK;
}

RecordTally NeedleDamage::tally() const {
    RecordTally t;
    t.off = spans_.as<int64_t>();
    t.end = t.off + n_;
    t.n = n_;
    t.damaged = counters_.as<unsigned long long>();
    t.uncorrectable = t.damaged + n_;
    t.unowned = t.damaged + 2 * n_;
    t.mask = masks_.as<unsigned>();
    return t;
}

int NeedleDamage::collect(swec_needle_damage* recs, uint64_t unowned[2]) {
    std::vector<unsigned long long> c;
    std::vector<unsigned> mask;
    SWEC_CUDA(counters_.read(&c));
    SWEC_CUDA(masks_.read(&mask));
    for (int j = 0; j < n_; j++) {
        swec_needle_damage& r = recs[order_[size_t(j)]];
        r.damaged_bytes = c[size_t(j)];
        r.uncorrectable_bytes = c[size_t(n_ + j)];
        r.shard_mask = mask[size_t(j)];
    }
    unowned[0] = c[size_t(2 * n_)];
    unowned[1] = c[size_t(2 * n_ + 1)];
    return SWEC_OK;
}

}  // namespace swec

using namespace swec;

extern "C" {

// Per 256 MiB piece: the shards copied to scratch, the parity re-encoded and the correcting locate run on the copy (its
// report is the one the locate call gives), the corrected data re-encoded, then the attribution against the caller's
// data shards, which are never written.
int swec_locate_needle_damage_device(swec_encoder* e, const void* const* shards, size_t n, int64_t dat_size, int64_t large,
                                     int64_t small, int radius, swec_needle_damage* records, int n_records,
                                     swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges,
                                     uint64_t unowned[2], void* stream) {
    int rc = check_needle_damage_args(0, nullptr, unowned, n_records, records);
    if (rc) return rc;
    if (!e || !shards) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    const DamageOut out{report, ranges, ranges_cap, n_ranges};
    if ((rc = out.check()) || (rc = check_radius(radius, 1, e->m))) return rc;
    if (dat_size < 0 || large <= 0 || small <= 0) return fail(SWEC_ERR_INVALID_ARG, "bad geometry");
    const int k = e->k, m = e->m;
    for (int i = 0; i < k + m; i++)
        if (!shards[i]) return fail(SWEC_ERR_INVALID_ARG, "NULL shard");
    const uint8_t* const* sh = reinterpret_cast<const uint8_t* const*>(shards);
    std::lock_guard<std::mutex> lock(e->mu);
    if ((rc = e->ensure_device())) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const Matrix rows = parity_rows(e);
    const size_t piece = std::min(n, size_t(256) << 20);
    DamageLocator locator;
    NeedleDamage nd;
    if ((rc = locator.init(rows, int64_t(n), radius, s, /*correct=*/true))) return rc;
    if ((rc = nd.init(k, m, StripeMap::encode(dat_size, k, large, small), records, n_records, 3, 0, 0, s))) return rc;
    StreamScratch scratch(s);
    if (piece) SWEC_CUDA(scratch.alloc(size_t(k + 2 * m) * piece));
    for (size_t off = 0; off < n; off += piece) {
        const size_t len = std::min(piece, n - off);
        const uint8_t* orig[SWEC_MAX_SHARDS];
        const uint8_t* data[SWEC_MAX_SHARDS];
        uint8_t* work[SWEC_MAX_SHARDS];
        uint8_t* comp[SWEC_MAX_SHARDS];
        for (int i = 0; i < k + m; i++) {
            work[i] = scratch.as<uint8_t>() + size_t(i) * piece;
            SWEC_CUDA(cudaMemcpyAsync(work[i], sh[i] + off, len, cudaMemcpyDeviceToDevice, s));
        }
        for (int i = 0; i < k; i++) {
            orig[i] = sh[i] + off;
            data[i] = work[i];
        }
        for (int q = 0; q < m; q++) comp[q] = scratch.as<uint8_t>() + size_t(k + m + q) * piece;
        if ((rc = e->apply(rows, data, comp, len, Layout{}, s))) return rc;
        if ((rc = locator.launch(comp, work, len, int64_t(off), s))) return rc;
        if ((rc = e->apply(rows, data, comp, len, Layout{}, s))) return rc;
        if ((rc = nd.launch(orig, work, comp, len, int64_t(off), 0, s))) return rc;
    }
    SWEC_CUDA(cudaStreamSynchronize(s));
    if ((rc = locator.collect(out))) return rc;
    return nd.collect(records, unowned);
}

}  // extern "C"
