// seaweedfs_b200/csrc/damage.cu — locate the wrong shard of every byte column whose parity does not match.
//
// For a column c = [d | p] of a shard set, computed parity XOR stored parity is the syndrome s = [P | I]·e of the
// error pattern e, so it is zero on a clean column and names the damage otherwise.  RS(k,m) has distance m+1: radius t
// decoding (2t <= m) blames exactly the wrong shards of a column with at most t of them, reports a column with t+1 ..
// m-t of them as uncorrectable, and may blame the wrong shards beyond that (include/swec.h states the guarantee).
//
//   swec_locate_kernel   grid-stride over 16-byte vectors of the 2m parity streams.  Clean vectors (the fast path)
//                        cost the loads, one OR per stream and one warp vote.  A warp with a non-zero syndrome reloads
//                        it and decodes every damaged column against log/exp tables and the logs of P in shared memory:
//                          one shard   exactly one non-zero component p: parity shard k+p; all m non-zero and
//                                      log s_i - log P[i][j] equal for every i: data shard j
//                          two shards  two non-zero components: those two parity shards; a data shard j and parity
//                                      shard k+p: the rows other than p are a multiple of P[:,j]; data shards a < b:
//                                      rows 0 and 1 solved by Cramer's rule, the other rows checked
//                        Per-lane runs (set, count, first, last) merge the columns a lane blames on one shard, and a
//                        warp merges equal runs with __match_any_sync / __reduce_*_sync before one set of atomics.
//                        Bytes after the last whole vector, and unaligned streams, go through a byte loop.
//                        The correcting instantiation (kCorrect) also XORs each blamed shard's error value into that
//                        shard's byte of the column, which makes the column a codeword again; it reads stored parity
//                        with coherent loads, because it writes it.
//                        The rebuilding instantiation (kRebuild) decodes the punctured code of a set with f missing
//                        shards: positions [0, k) are the first k present shards (the information set I), positions
//                        [k, k+c) the other present ones, whose rows P' = G[C]·G[I]^-1 take the place of P.  The f
//                        rebuilt streams were computed from I by the rows R = G[missing]·G[I]^-1, so an error e_j in
//                        information position j put R[r][j]·e_j into rebuilt byte x of stream r: the kernel XORs it
//                        back out.  A blamed check position, and every present shard, are left as they are.  Radius 0
//                        counts every damaged column as uncorrectable and decodes none.
//                        The decoding instantiation (kDecode) is kRebuild for ec.decode: its rows are those of the
//                        missing data shards and the check shards only, and it also XORs each located error value of an
//                        information position that holds a data shard into that shard's own byte, so every data byte of
//                        a column decoded within the radius is the true one.  Present parity shards are never written.
// The column decoder (decode_column) lives in locate_decode.cuh, which the page decode of the sketch calls shares.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "damage.h"
#include "device_common.cuh"
#include "engine.h"
#include "locate_decode.cuh"

namespace swec {

namespace {

constexpr int kSets = SWEC_MAX_SHARDS + 1;  // one counter set per shard, and one for uncorrectable columns (set k+m)
constexpr int kCounters = 3 * kSets + 1;    // bytes[kSets], first[kSets], last[kSets], damaged columns
constexpr int kPageShift = 12;              // 4 KiB pages

enum : int { kLocate = 0, kCorrect = 1, kRebuild = 2, kDecode = 3 };  // the instantiations of swec_locate_kernel


// kRebuild and kDecode only, in shared memory of its own so that the other instantiations copy no more than before
struct RebuildTables {
    u8 logr[kLogRBytes];  // CheckedPlan::rebuilt_logs
};
constexpr int kRebuildWords = int(sizeof(RebuildTables) / 4);

struct LocateParams {
    const u8* comp[SWEC_MAX_SHARDS];
    const u8* stored[SWEC_MAX_SHARDS];
    u64 n, base;
    int k, m, radius;
    const u32* tables;
    unsigned long long* ctr;
    u32* pages;
    u64 page_words;
    u8* fix[SWEC_MAX_SHARDS];  // kCorrect: the k+m shards' bytes of these columns (fix[k+p] == stored[p]);
                               // kRebuild: the nout rebuilt streams; kDecode: those, then at fix[nout + j] the bytes of
                               // information position j when it holds a data shard (NULL for a parity shard)
    int nout;                  // kRebuild, kDecode: rebuilt streams
    const u32* rtables;        // kRebuild, kDecode: RebuildTables
};

struct Run {  // columns one lane blamed on one set, in increasing offset order
    int set;  // valid while cnt > 0
    u32 cnt;
    u64 first, last;
};

__device__ __forceinline__ void set_page(const LocateParams& p, int set, u64 off) {
    const u64 page = off >> kPageShift;
    atomicOr(p.pages + u64(set) * p.page_words + (page >> 5), 1u << (page & 31));
}

// a run of one lane's columns: they lie within 16 bytes (or one byte), so in at most two pages
__device__ void flush_plain(const LocateParams& p, Run& r) {
    if (!r.cnt) return;
    atomicAdd(p.ctr + r.set, (unsigned long long)r.cnt);
    atomicMin(p.ctr + kSets + r.set, (unsigned long long)r.first);
    atomicMax(p.ctr + 2 * kSets + r.set, (unsigned long long)r.last);
    set_page(p, r.set, r.first);
    if ((r.last >> kPageShift) != (r.first >> kPageShift)) set_page(p, r.set, r.last);
    r.cnt = 0;
}

// Whole warp, converged.  The warp's columns lie within 512 bytes of wbase, so in at most two pages, and a set's
// first and last column are in both of them.
__device__ __forceinline__ void flush_warp(const LocateParams& p, Run& r, u64 wbase) {
    const int key = r.cnt ? r.set : -1;
    const u32 group = __match_any_sync(0xffffffffu, key);
    if (key < 0) return;
    const u32 cnt = __reduce_add_sync(group, r.cnt);
    const u32 lo = __reduce_min_sync(group, u32(r.first - wbase));
    const u32 hi = __reduce_max_sync(group, u32(r.last - wbase));
    r.cnt = 0;
    if ((threadIdx.x & 31) != u32(__ffs(group) - 1)) return;
    Run w{key, cnt, wbase + lo, wbase + hi};
    flush_plain(p, w);
}

__device__ __forceinline__ void record(const LocateParams& p, Run* run, int set, u64 off) {
    int i;
    if (run[0].cnt && run[0].set == set) i = 0;
    else if (run[1].cnt && run[1].set == set) i = 1;
    else if (!run[0].cnt) i = 0;
    else {
        flush_plain(p, run[1]);  // a third set within one lane's columns: rare
        i = 1;
    }
    if (!run[i].cnt) {
        run[i].set = set;
        run[i].first = off;
    }
    run[i].cnt++;
    run[i].last = off;
}

// kRebuild: the error value e of position j carried into byte x of every rebuilt stream (nothing for a check position)
__device__ __forceinline__ void propagate(const LocateParams& p, const LocateTables& t, const u8* logr, int j, u8 e, u64 x) {
    if (j >= p.k) return;
    const int le = t.log[e];
    for (int r = 0; r < p.nout; r++) {
        const u8 lr = logr[r * 32 + j];
        if (lr != kLogZero) p.fix[r][x] ^= t.exp[lr + le];
    }
}

// kDecode: the error value e of information position j XORed into its own byte, when it holds a data shard
__device__ __forceinline__ void restore(const LocateParams& p, int j, u8 e, u64 x) {
    if (j >= p.k) return;
    if (u8* d = p.fix[p.nout + j]) d[x] ^= e;
}

// column x of the launch (shard offset p.base + x); the correcting kernel XORs the error values into the shards, the
// rebuilding kernel their images into the rebuilt streams, the decoding kernel both into the data shards
template <int MODE>
__device__ __forceinline__ void blame(const LocateParams& p, const LocateTables& t, const u8* logr, const u8* s, int m,
                                      u64 x, Run* run) {
    int a = -1, b = -1;
    u8 ea = 0, eb = 0;
    const u64 off = p.base + x;
    const int found = ((MODE == kRebuild || MODE == kDecode) && p.radius == 0)
                          ? 0
                          : decode_column<MODE != kLocate>(t, s, p.k, m, p.radius, &a, &b, &ea, &eb);
    if (!found) {
        record(p, run, p.k + m, off);
        return;
    }
    record(p, run, a, off);
    if (MODE == kCorrect) p.fix[a][x] ^= ea;
    if (MODE == kRebuild || MODE == kDecode) propagate(p, t, logr, a, ea, x);
    if (MODE == kDecode) restore(p, a, ea, x);
    if (found == 2) {
        record(p, run, b, off);
        if (MODE == kCorrect) p.fix[b][x] ^= eb;
        if (MODE == kRebuild || MODE == kDecode) propagate(p, t, logr, b, eb, x);
        if (MODE == kDecode) restore(p, b, eb, x);
    }
}

// Stored parity is read through the non-coherent path only by the kernels that do not write it.
template <bool CORRECT>
__device__ __forceinline__ uint4 load_stored(const u8* p) {
    if (CORRECT) return *reinterpret_cast<const uint4*>(p);
    return swec_ldg_stream(p);
}

__device__ __forceinline__ u8 byte_of(const uint4& x, int c) {
    const u32 w = c < 4 ? x.x : c < 8 ? x.y : c < 12 ? x.z : x.w;
    return u8(w >> ((c & 3) * 8));
}

__device__ __forceinline__ uint4 xor4(const uint4& a, const uint4& b) {
    return make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w);
}

// MT > 0: m known at compile time; 0: run-time m.  MODE: kLocate, kCorrect (fix every column decoded within the radius
// in place), kRebuild (take the errors of the information positions out of the rebuilt streams) or kDecode (kRebuild,
// and the errors of the information positions that hold data shards corrected in place too).  A column's bytes
// are read and written only by the thread that owns its vector (or its byte in the tail loop).
template <int MT, int MODE>
__global__ void __launch_bounds__(256) swec_locate_kernel(const __grid_constant__ LocateParams p) {
    constexpr bool CORRECT = MODE == kCorrect;
    __shared__ __align__(16) u32 words[kTableWords];
    for (int i = threadIdx.x; i < kTableWords; i += blockDim.x) words[i] = p.tables[i];
    const u8* logr = nullptr;
    if constexpr (MODE == kRebuild || MODE == kDecode) {
        __shared__ __align__(16) u32 rwords[kRebuildWords];
        for (int i = threadIdx.x; i < kRebuildWords; i += blockDim.x) rwords[i] = p.rtables[i];
        logr = reinterpret_cast<const u8*>(rwords);
    }
    __syncthreads();
    const LocateTables& t = *reinterpret_cast<const LocateTables*>(words);
    constexpr int kMaxM = MT > 0 ? MT : SWEC_MAX_SHARDS;
    const int m = MT > 0 ? MT : p.m;
    unsigned long long align = 0;
    for (int i = 0; i < m; i++)
        align |= reinterpret_cast<unsigned long long>(p.comp[i]) | reinterpret_cast<unsigned long long>(p.stored[i]);
    const u64 nvec = (align & 15) == 0 ? p.n >> 4 : 0;
    const u32 lane = threadIdx.x & 31;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    Run run[2] = {{-1, 0, 0, 0}, {-1, 0, 0, 0}};

    // vb is the first vector of this warp: every lane of a warp takes the same number of turns
    for (u64 vb = (u64)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); vb < nvec; vb += stride) {
        const u64 v = vb + lane;
        u32 diff = 0;
        if (v < nvec) {
#pragma unroll
            for (int i = 0; i < kMaxM; i++) {
                if (MT == 0 && i >= m) break;
                const uint4 d = xor4(swec_ldg_stream(p.comp[i] + (v << 4)), load_stored<CORRECT>(p.stored[i] + (v << 4)));
                diff |= d.x | d.y | d.z | d.w;
            }
        }
        if (!__any_sync(0xffffffffu, diff != 0)) continue;
        u32 damaged = 0;
        if (diff) {
            uint4 x[kMaxM];
            for (int i = 0; i < m; i++)
                x[i] = xor4(__ldg(reinterpret_cast<const uint4*>(p.comp[i]) + v),
                            CORRECT ? reinterpret_cast<const uint4*>(p.stored[i])[v]
                                    : __ldg(reinterpret_cast<const uint4*>(p.stored[i]) + v));
            for (int c = 0; c < 16; c++) {
                u8 s[kMaxM];
                u8 any = 0;
                for (int i = 0; i < m; i++) {
                    s[i] = byte_of(x[i], c);
                    any |= s[i];
                }
                if (!any) continue;
                damaged++;
                blame<MODE>(p, t, logr, s, m, (v << 4) + u64(c), run);
            }
        }
        const u64 wbase = p.base + (vb << 4);
        flush_warp(p, run[0], wbase);
        flush_warp(p, run[1], wbase);
        damaged = __reduce_add_sync(0xffffffffu, damaged);
        if (lane == 0 && damaged) atomicAdd(p.ctr + 3 * kSets, (unsigned long long)damaged);
    }

    for (u64 x = (nvec << 4) + (u64)blockIdx.x * blockDim.x + threadIdx.x; x < p.n; x += stride) {
        u8 s[kMaxM];
        u8 any = 0;
        for (int i = 0; i < m; i++) {
            s[i] = p.comp[i][x] ^ p.stored[i][x];
            any |= s[i];
        }
        if (!any) continue;
        atomicAdd(p.ctr + 3 * kSets, 1ull);
        blame<MODE>(p, t, logr, s, m, x, run);
        flush_plain(p, run[0]);
        flush_plain(p, run[1]);
    }
}

template <int MT, int MODE>
unsigned locate_grid(u64 n) {
    static const int per_sm = [] {  // resident CTAs per SM, the same on every device of this architecture
        int c = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, swec_locate_kernel<MT, MODE>, 256, 0) != cudaSuccess) {
            cudaGetLastError();
            c = 4;
        }
        return std::max(1, c);
    }();
    return grid_cap((n / 16 + 255) / 256 + 1, per_sm);
}

// The instantiation for m among the compiled-in MT values of MODE, else the run-time m one (MT = 0).
template <int MODE, int MT = 0, int... MORE>
void launch_locate(int m, const LocateParams& p, u64 n, cudaStream_t s) {
    if constexpr (MT != 0) {
        if (m != MT) return launch_locate<MODE, MORE...>(m, p, n, s);
    }
    swec_locate_kernel<MT, MODE><<<locate_grid<MT, MODE>(n), 256, 0, s>>>(p);
}

}  // namespace

int DamageOut::check() const {
    if (!report) return fail(SWEC_ERR_INVALID_ARG, "report is NULL");
    if (cap < 0 || (cap > 0 && !ranges))
        return fail(SWEC_ERR_INVALID_ARG, "ranges_cap must be >= 0, and ranges non-NULL when it is > 0");
    return SWEC_OK;
}

void DamageOut::unchecked() const {
    memset(report, 0, sizeof *report);
    report->first_uncorrectable = report->last_uncorrectable = -1;
    for (int i = 0; i < SWEC_MAX_SHARDS; i++) report->shard_first[i] = report->shard_last[i] = -1;
    if (n_ranges) *n_ranges = 0;
}

int check_radius(int radius, int lowest, int m) {
    if (radius < lowest || radius > 2)
        return fail(SWEC_ERR_INVALID_ARG, lowest ? "radius must be 1 or 2" : "radius must be 0, 1 or 2");
    if (m < 2 * radius)
        return fail(SWEC_ERR_INVALID_ARG, "radius " + std::to_string(radius) + " needs at least " +
                                              std::to_string(2 * radius) + " parity shards, the code has " + std::to_string(m));
    return SWEC_OK;
}

bool CheckedPlan::build(const Matrix& gen, int k, const uint8_t* present, bool decode) {
    this->decode = decode;
    std::vector<uint8_t> mask(size_t(gen.rows), 0);  // the information set alone: every other shard gets a row
    for (int i = 0, n = 0; i < gen.rows && n < k; i++)
        if (present[i]) mask[size_t(i)] = 1, n++;
    std::vector<int> all;
    Matrix rows;
    if (!rs_reconstruct_plan(gen, k, mask.data(), false, &info, &all, &rows)) return false;
    outs.clear();
    fused = Matrix(0, k);
    check_rows.clear();
    rebuilt_rows.clear();
    for (size_t o = 0; o < all.size(); o++) {
        const int id = all[o];
        if (decode && id >= k && !present[id]) continue;  // a missing parity shard
        (present[id] ? check_rows : rebuilt_rows).push_back(int(outs.size()));
        outs.push_back(id);
        fused.v.insert(fused.v.end(), rows.row(int(o)), rows.row(int(o)) + k);
        fused.rows++;
    }
    return true;
}

CheckedPlan CheckedPlan::all_present(const Matrix& gen, int k) {
    const std::vector<uint8_t> all(size_t(gen.rows), 1);
    CheckedPlan plan;
    plan.build(gen, k, all.data(), false);
    return plan;
}

int CheckedPlan::position(int id) const {
    const int k = int(info.size()), c = this->c();
    for (int j = 0; j < k; j++)
        if (info[size_t(j)] == id) return j;
    for (int i = 0; i < c; i++)
        if (check(i) == id) return k + i;
    for (size_t o = 0; o < outs.size(); o++)
        if (outs[o] == id) return k + c + int(o);
    return -1;
}

Matrix CheckedPlan::checks() const {
    const int k = fused.cols;
    Matrix pc(c(), k);
    for (int i = 0; i < c(); i++)
        for (int j = 0; j < k; j++) pc.at(i, j) = fused.at(check_rows[size_t(i)], j);
    return pc;
}

void CheckedPlan::rebuilt_logs(uint8_t* logr) const {
    u8 log[256], exp[512];
    log_exp_tables(log, exp);
    memset(logr, kLogZero, kLogRBytes);
    for (size_t r = 0; r < rebuilt_rows.size(); r++)
        for (int j = 0; j < fused.cols; j++)
            if (const u8 v = fused.at(rebuilt_rows[r], j)) logr[r * 32 + size_t(j)] = log[v];
}

int DamageLocator::init(const Matrix& parity, int64_t shard_len, int radius, cudaStream_t s, bool correct) {
    k_ = parity.cols;
    m_ = parity.rows;
    radius_ = radius;
    correct_ = correct;
    shard_len_ = shard_len;
    ids_.resize(size_t(k_ + m_));
    for (int i = 0; i < k_ + m_; i++) ids_[size_t(i)] = i;
    LocateTables t;
    locate_tables(parity, &t);
    const int64_t pages = (shard_len + (int64_t(1) << kPageShift) - 1) >> kPageShift;
    page_words_ = std::max<size_t>(1, size_t((pages + 31) / 32));
    const size_t page_bytes = size_t(k_ + m_ + 1) * page_words_ * 4;
    SWEC_CUDA(counters_.alloc(kCounters * sizeof(unsigned long long)));
    SWEC_CUDA(pages_.alloc(page_bytes));
    unsigned long long* ctr = counters_.as<unsigned long long>();
    SWEC_CUDA(cudaMemsetAsync(ctr, 0, kCounters * sizeof(unsigned long long), s));
    SWEC_CUDA(cudaMemsetAsync(ctr + kSets, 0xff, kSets * sizeof(unsigned long long), s));  // first = max
    SWEC_CUDA(cudaMemsetAsync(pages_.as<void>(), 0, page_bytes, s));
    SWEC_CUDA(tables_.upload(&t, 1, s));  // synchronises s, after the clears
    return SWEC_OK;
}

int DamageLocator::init_rebuild(const CheckedPlan& plan, int64_t shard_len, int radius, cudaStream_t s) {
    if (int rc = init(plan.checks(), shard_len, plan.radius(radius), s)) return rc;
    rebuild_ = true;
    decode_ = plan.decode;
    check_rows_ = plan.check_rows;
    out_rows_ = plan.rebuilt_rows;
    for (int j = 0; j < k_; j++) ids_[size_t(j)] = plan.info[size_t(j)];
    for (int i = 0; i < m_; i++) ids_[size_t(k_ + i)] = plan.check(i);
    RebuildTables rt;
    plan.rebuilt_logs(rt.logr);
    SWEC_CUDA(rtables_.upload(&rt, 1, s));
    return SWEC_OK;
}

int DamageLocator::launch(uint8_t* const* computed, uint8_t* const* shards, size_t n, int64_t base, cudaStream_t s) {
    if (n == 0) return SWEC_OK;
    LocateParams p;
    memset(&p, 0, sizeof p);
    for (int i = 0; i < m_; i++) {
        p.comp[i] = computed[rebuild_ ? check_rows_[size_t(i)] : i];
        p.stored[i] = shards[k_ + i];
    }
    if (correct_)
        for (int i = 0; i < k_ + m_; i++) p.fix[i] = shards[i];
    if (rebuild_) {
        for (size_t r = 0; r < out_rows_.size(); r++) p.fix[r] = computed[out_rows_[r]];
        p.nout = int(out_rows_.size());
        p.rtables = rtables_.as<u32>();
    }
    if (decode_)  // nout + k <= k + m slots: the rebuilt streams are missing data shards
        for (int j = 0; j < k_; j++) p.fix[p.nout + j] = ids_[size_t(j)] < k_ ? shards[j] : nullptr;
    p.n = n;
    p.base = u64(base);
    p.k = k_;
    p.m = m_;
    p.radius = radius_;
    p.tables = tables_.as<u32>();
    p.ctr = counters_.as<unsigned long long>();
    p.pages = pages_.as<u32>();
    p.page_words = page_words_;
    if (decode_) launch_locate<kDecode, 4, 3>(m_, p, n, s);
    else if (rebuild_) launch_locate<kRebuild, 3>(m_, p, n, s);
    else if (correct_) launch_locate<kCorrect, 4>(m_, p, n, s);
    else launch_locate<kLocate, 4>(m_, p, n, s);
    SWEC_CUDA(launched());
    return SWEC_OK;
}

int DamageLocator::collect(const DamageOut& out, std::vector<swec_damage_range>* all) {
    const int n = k_ + m_;
    std::vector<unsigned long long> c;
    std::vector<uint32_t> bits;  // n + 1 page bitmaps
    SWEC_CUDA(counters_.read(&c));
    SWEC_CUDA(pages_.read(&bits));
    swec_damage_report* report = out.report;
    out.unchecked();
    report->columns = uint64_t(shard_len_);
    report->damaged_columns = c[3 * kSets];
    report->uncorrectable_columns = c[size_t(n)];
    report->first_uncorrectable = c[size_t(n)] ? int64_t(c[size_t(kSets + n)]) : -1;
    report->last_uncorrectable = c[size_t(n)] ? int64_t(c[size_t(2 * kSets + n)]) : -1;
    for (int i = 0; i < n; i++) {  // kernel position i is shard ids_[i]
        if (!c[size_t(i)]) continue;
        const int id = ids_[size_t(i)];
        report->shard_bytes[id] = c[size_t(i)];
        report->shard_first[id] = int64_t(c[size_t(kSets + i)]);
        report->shard_last[id] = int64_t(c[size_t(2 * kSets + i)]);
    }
    // maximal runs of flagged pages: shards in ascending id (ids_ ascends), then the uncorrectable columns
    const int64_t pages = (shard_len_ + (int64_t(1) << kPageShift) - 1) >> kPageShift;
    int total = 0;
    if (all) all->clear();
    for (int set = 0; set <= n; set++) {
        const uint32_t* w = bits.data() + size_t(set) * page_words_;
        auto flagged = [&](int64_t pg) { return (w[pg >> 5] >> (pg & 31)) & 1u; };
        for (int64_t pg = 0; pg < pages;) {
            if ((pg & 31) == 0 && w[pg >> 5] == 0) {
                pg += 32;
                continue;
            }
            if (!flagged(pg)) {
                pg++;
                continue;
            }
            int64_t end = pg + 1;
            while (end < pages && flagged(end)) end++;
            swec_damage_range r;
            r.shard_id = set < n ? ids_[size_t(set)] : -1;
            r.reserved = 0;
            r.offset = pg << kPageShift;
            r.length = std::min(end << kPageShift, shard_len_) - r.offset;
            if (total < out.cap) out.ranges[total] = r;
            if (all) all->push_back(r);
            total++;
            pg = end;
        }
    }
    if (out.n_ranges) *out.n_ranges = total;
    return SWEC_OK;
}

}  // namespace swec
