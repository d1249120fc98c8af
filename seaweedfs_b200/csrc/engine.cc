// seaweedfs_b200/csrc/engine.cc — encoder object, matrix→kernel dispatch, host staging pipeline.
#include "engine.h"
#include "damage.h"
#include "io_pool.h"
#include "volume_format.h"

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <thread>

#include <execinfo.h>
#include <signal.h>
#include <sys/mman.h>
#include <unistd.h>

namespace swec {

// ------------------------------------------------------------------ crash diagnostics (SWEC_DEBUG_SEGV=1)
static void segv_backtrace(int sig) {
    void* frames[64];
    const int n = backtrace(frames, 64);
    const char msg[] = "\n[swec] fatal signal, backtrace:\n";
    if (write(2, msg, sizeof msg - 1) < 0) {}
    backtrace_symbols_fd(frames, n, 2);
    signal(sig, SIG_DFL);
    raise(sig);
}
static const int g_segv_hook = [] {
    if (getenv("SWEC_DEBUG_SEGV")) {
        signal(SIGSEGV, segv_backtrace);
        signal(SIGABRT, segv_backtrace);
        signal(SIGBUS, segv_backtrace);
        // Python's faulthandler restores the default handlers when the interpreter finalises; hook
        // again once exit() starts running handlers so crashes in static destructors are seen too
        std::atexit([] {
            signal(SIGSEGV, segv_backtrace);
            signal(SIGABRT, segv_backtrace);
            const char m[] = "[swec] exit handlers running\n";
            if (write(2, m, sizeof m - 1) < 0) {}
        });
    }
    return 0;
}();

// ------------------------------------------------------------------ errors

static thread_local std::string t_last_error;

void set_last_error(const std::string& msg) { t_last_error = msg; }
const char* last_error() { return t_last_error.c_str(); }

int fail(int status, const std::string& msg) {
    set_last_error(msg);
    return status;
}

int cuda_fail(cudaError_t e, const char* what) {
    const bool nodev = e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInvalidDevice;
    set_last_error(std::string(what) + ": " + cudaGetErrorName(e) + " — " + cudaGetErrorString(e));
    return nodev ? SWEC_ERR_NO_DEVICE : SWEC_ERR_CUDA;
}

size_t env_size(const char* name, size_t dflt) {
    const char* e = getenv(name);
    if (!e || !*e) return dflt;
    const long long v = atoll(e);
    return v > 0 ? size_t(v) : dflt;
}

std::atomic<long> g_opt_stage_chunk{long(env_size("SWEC_STAGE_CHUNK", size_t(16) << 20))};
std::atomic<long> g_opt_stage_slots{long(env_size("SWEC_STAGE_SLOTS", 3))};
size_t stage_slots() { return size_t(std::max(2l, g_opt_stage_slots.load())); }
// Encoder-seam calls (swec_encode & co. on host buffers) are cut into at least this many pieces — never smaller
// than host_min_chunk — so that the bounce copy / H2D of piece c+1, the kernel of piece c and the D2H / copy-back of
// piece c-1 overlap INSIDE one call: the Go call sites hand over 256 KiB (encodeDataOneBatch) or 1 MiB
// (rebuildEcFiles) per shard and wait for the result.
std::atomic<long> g_opt_host_pieces{long(env_size("SWEC_HOST_PIECES", 4))};
std::atomic<long> g_opt_host_min_chunk{long(env_size("SWEC_HOST_MIN_CHUNK", size_t(256) << 10))};
// Zero-copy at the Encoder seam: the kernel reads the (mapped, pinned) host shards over PCIe itself and writes the
// parity straight back to host memory — no staging in HBM, no DMA enqueue, one launch per piece.  What a short
// synchronous call costs is API round trips, not bytes: 0 = never, 1 = whenever the buffers allow it,
// 2 = auto: calls of at most host_zero_copy_max bytes per shard (bigger ones stream through the DMA ring).
// The 2 MiB threshold was chosen on an earlier GPU generation (zero-copy ahead up to ~1-2 MiB per shard, the 4-piece
// DMA ring from 4 MiB); not yet re-measured on the H100 (scripts/bench_host_api.py sweeps it).
std::atomic<long> g_opt_host_zero_copy{long(env_size("SWEC_HOST_ZERO_COPY", 2))};
std::atomic<long> g_opt_host_zero_copy_max{long(env_size("SWEC_HOST_ZERO_COPY_MAX", size_t(2) << 20))};
std::atomic<long> g_opt_host_copy_spin_us{long(env_size("SWEC_HOST_COPY_SPIN_US", 200))};
std::atomic<long> g_opt_host_copy_threads{long(env_size("SWEC_HOST_COPY_THREADS", 0))};  // 0 = auto
std::atomic<long> g_opt_file_direct_io{long(env_size("SWEC_FILE_DIRECT", 0)) & 3};
std::atomic<long> g_opt_jit_enabled{1};
std::atomic<long> g_opt_jit_min_bytes{long(env_size("SWEC_JIT_MIN_BYTES", size_t(64) << 20))};

// ------------------------------------------------------------------ encoder lifetime

swec_encoder_impl::~swec_encoder_impl() {
    if (device < 0) return;
    if (cudaSetDevice(device) != cudaSuccess) return;
    for (auto& kv : tables) {
        cudaFree(kv.second.compact);
        cudaFree(kv.second.replicated);
    }
    ring.release();
    if (stream) cudaStreamDestroy(stream);
}

int swec_encoder_impl::ensure_device() {
    if (device < 0) return fail(SWEC_ERR_NO_DEVICE, "encoder was created without a device (device < 0); no CPU fallback exists");
    SWEC_CUDA(cudaSetDevice(device));
    if (!stream) SWEC_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    return SWEC_OK;
}

int swec_encoder_impl::ensure_slots(size_t chunk) {
    const size_t nslots = stage_slots(), streams = size_t(k) + 2 * size_t(m);
    const size_t have = slot_chunk();
    if (ring.slots.size() == nslots && have >= chunk) return SWEC_OK;
    // grow geometrically (callers with varying sizes must not re-pin memory on every larger call)
    if (!ring.slots.empty() && have < chunk)
        chunk = std::min(std::max(chunk, 2 * have), std::max(chunk, size_t(g_opt_stage_chunk.load())));
    chunk = std::max<size_t>(chunk, 64 * 1024);
    return ring.allocate(device, nslots, streams * chunk);
}

// ------------------------------------------------------------------ tables

static std::vector<uint8_t> matrix_key(const Matrix& rows) {
    std::vector<uint8_t> key{uint8_t(rows.rows), uint8_t(rows.cols)};
    key.insert(key.end(), rows.v.begin(), rows.v.end());
    return key;
}

int swec_encoder_impl::get_tables(const Matrix& rows, DeviceTables* out, cudaStream_t s) {
    const auto key = matrix_key(rows);
    auto it = tables.find(key);
    if (it != tables.end()) {
        *out = it->second;
        return SWEC_OK;
    }
    const GF& gf = GF::get();
    const int K = rows.cols, R = rows.rows;
    std::vector<u32> compact(size_t(K) * 32), repl(size_t(K) * 32 * 32);
    for (int i = 0; i < K; i++)
        for (int h = 0; h < 2; h++)
            for (int v = 0; v < 16; v++) {
                u32 w = 0;
                for (int r = 0; r < R; r++) w |= u32(gf.mul[rows.at(r, i)][uint8_t(v << (4 * h))]) << (8 * r);
                const size_t e = size_t(i) * 32 + size_t(h) * 16 + size_t(v);
                compact[e] = w;
                for (int lane = 0; lane < 32; lane++) repl[e * 32 + size_t(lane)] = w;
            }
    DeviceTables t;
    SWEC_CUDA(cudaMalloc(reinterpret_cast<void**>(&t.compact), compact.size() * 4));
    SWEC_CUDA(cudaMalloc(reinterpret_cast<void**>(&t.replicated), repl.size() * 4));
    // synchronous copies from pageable memory: the vectors die at return
    SWEC_CUDA(cudaMemcpyAsync(t.compact, compact.data(), compact.size() * 4, cudaMemcpyHostToDevice, s));
    SWEC_CUDA(cudaMemcpyAsync(t.replicated, repl.data(), repl.size() * 4, cudaMemcpyHostToDevice, s));
    SWEC_CUDA(cudaStreamSynchronize(s));
    tables[key] = t;
    *out = t;
    return SWEC_OK;
}

// ------------------------------------------------------------------ matrix → kernel dispatch

static bool is_rs10x4_parity(const swec_encoder_impl& e, const Matrix& rows) {
    if (!e.rs10x4 || rows.rows != 4 || rows.cols != 10 || !g_opt_use_aot.load()) return false;
    for (int r = 0; r < 4; r++)
        if (memcmp(rows.row(r), e.gen.row(10 + r), 10) != 0) return false;
    return true;
}

static int ilog2_exact(uint64_t v) {
    if (!v || (v & (v - 1))) return -1;
    int s = 0;
    while ((v >> s) != 1) s++;
    return s;
}

int swec_encoder_impl::apply(const Matrix& rows, const uint8_t* const* in, uint8_t* const* out, size_t n,
                             const Layout& layout, cudaStream_t s) {
    const int R = rows.rows, K = rows.cols;
    if (R == 0 || n == 0) return SWEC_OK;
    if (K > SWEC_MAX_INPUTS) return fail(SWEC_ERR_INVALID_ARG, "too many input shards");

    uintptr_t align = 0;
    for (int i = 0; i < K; i++) align |= reinterpret_cast<uintptr_t>(in[i]);
    for (int r = 0; r < R; r++) align |= reinterpret_cast<uintptr_t>(out[r]);
    if (layout.blocked) align |= layout.block_bytes;
    const bool aligned = (align & 15) == 0;
    const size_t nvec = aligned ? n / 16 : 0;
    const size_t tail_off = nvec * 16, tail = n - tail_off;
    if (layout.blocked && (!aligned || tail))
        return fail(SWEC_ERR_INVALID_ARG, "blocked layout needs 16-byte aligned blocks");

    auto fill = [&](SwecApplyParams& p, int r0, int rn, size_t off) {
        memset(&p, 0, sizeof p);
        for (int i = 0; i < K; i++) p.in[i] = in[i] + off;
        for (int r = 0; r < rn; r++) p.out[r] = out[r0 + r] + off;
        p.nvec = nvec;
        p.block_shift = -1;
        if (layout.blocked) {
            p.block_vecs = layout.block_bytes / 16;
            p.block_shift = ilog2_exact(p.block_vecs);
            p.row_extra = uint64_t(K - 1) * layout.block_bytes;
        }
    };

    if (nvec) {
        SwecApplyParams p;
        if (is_rs10x4_parity(*this, rows)) {
            fill(p, 0, R, 0);
            SWEC_CUDA(launch_rs10x4_encode(p, layout.blocked, s));
        } else if (const int aot = (rs10x4 && !layout.blocked && R <= 4 && K == 10 && g_opt_use_aot.load()) ? aot_recon_find(R, K, rows.v.data()) : -1;
                   aot >= 0) {
            // one of the reconstruct matrices compiled with the library (any single-shard loss, shards 0-3 lost):
            // no compile, no threshold — needle-sized degraded reads take the Horner kernel too
            fill(p, 0, R, 0);
            SWEC_CUDA(launch_aot_recon(aot, p, s));
        } else {
            // specialised (NVRTC) Horner kernel when the stream is long enough to pay for the
            // compile, or the kernel is already cached; otherwise shared-memory tables.
            // Long streams compile the specialised kernel inline (≈0.3 s, amortised); short ones start
            // the compile in the background, are served from the table kernel meanwhile, and pick the
            // fast kernel up once it is ready (degraded reads repeat the same few matrices).
            const size_t jit_min = size_t(g_opt_jit_min_bytes.load());
            std::shared_ptr<JitKernel> jk;
            if (R <= SWEC_MAX_OUTPUTS && g_opt_jit_enabled.load() && jit_available()) {
                const bool wait = (size_t(K) * n >= jit_min && !never_wait_for_jit) || layout.blocked;
                const int rc = jit_get(this, rows, &jk, wait, /*hot=*/never_wait_for_jit);
                if (rc != SWEC_OK && getenv("SWEC_JIT_STRICT")) return rc;
            }
            if (jk) {
                fill(p, 0, R, 0);
                SWEC_CUDA(jit_launch(*jk, p, layout.blocked, s));
            } else {
                if (layout.blocked) return fail(SWEC_ERR_INVALID_ARG, "blocked layout needs a specialised kernel");
                for (int r0 = 0; r0 < R; r0 += 4) {
                    const int rn = std::min(4, R - r0);
                    Matrix sub(rn, K);
                    for (int r = 0; r < rn; r++) memcpy(&sub.v[size_t(r) * K], rows.row(r0 + r), size_t(K));
                    DeviceTables t;
                    int rc = get_tables(sub, &t, s);
                    if (rc) return rc;
                    fill(p, r0, rn, 0);
                    SWEC_CUDA(launch_table_apply(p, t.replicated, K, rn, s));
                }
            }
        }
    }
    if (tail) {
        for (int r0 = 0; r0 < R; r0 += 4) {
            const int rn = std::min(4, R - r0);
            Matrix sub(rn, K);
            for (int r = 0; r < rn; r++) memcpy(&sub.v[size_t(r) * K], rows.row(r0 + r), size_t(K));
            DeviceTables t;
            int rc = get_tables(sub, &t, s);
            if (rc) return rc;
            SwecApplyParams p;
            fill(p, r0, rn, tail_off);
            SWEC_CUDA(launch_bytes_apply(p, t.compact, K, rn, tail, s));
        }
    }
    return SWEC_OK;
}

// ------------------------------------------------------------------ host staging pipeline
// Chunks of every stream travel pinned-host → HBM → kernel → pinned-host on one of a few slots,
// each with its own stream, so H2D of chunk c+1, the kernel of chunk c and D2H of chunk c-1
// overlap.  Caller buffers that are already pinned (swec_alloc_pinned / cudaHostRegister) are
// DMA'd directly; pageable ones bounce through the slot's pinned buffer.

namespace {

struct DeviceCounter {
    unsigned long long* p = nullptr;
    ~DeviceCounter() {
        if (p) cudaFree(p);
    }
};

// *gpu_ptr: the address the GPU uses for this memory (device memory: itself; mapped pinned host memory: its device
// alias, the same value under unified addressing), nullptr if a kernel cannot reach it
bool is_pinned_or_device(const void* p, bool* is_device, const void** gpu_ptr = nullptr) {
    cudaPointerAttributes a;
    if (gpu_ptr) *gpu_ptr = nullptr;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        *is_device = false;
        return false;
    }
    *is_device = a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
    const bool direct = a.type == cudaMemoryTypeHost || *is_device;
    if (gpu_ptr && direct) *gpu_ptr = a.devicePointer;
    return direct;
}

}  // namespace

// ---- bounce copies between pageable caller memory and the pinned ring run across a few threads: one core moves
// ~10 GB/s, far less than a PCIe x16 link, so a single memcpy loop would be the whole cost of an Encoder-level call
// from Go heap memory.
namespace {

struct CopyJob {
    uint8_t* dst;
    const uint8_t* src;
    size_t len;
};

IoPool* host_pool() {  // leaked on purpose (threads must outlive static destructors); nullptr = copy inline
    static IoPool* pool = [] () -> IoPool* {
        long n = g_opt_host_copy_threads.load();
        if (n <= 0) n = std::min<long>(8, std::max<long>(2, long(std::thread::hardware_concurrency()) / 8));
        return n > 1 ? new IoPool(size_t(n - 1), unsigned(g_opt_host_copy_spin_us.load())) : nullptr;  // the caller takes a share too
    }();
    return pool;
}

void parallel_copy(const std::vector<CopyJob>& jobs) {
    constexpr size_t kPiece = size_t(128) << 10, kInlineBelow = size_t(256) << 10;
    size_t total = 0;
    for (const CopyJob& j : jobs) total += j.len;
    IoPool* pool = total > kInlineBelow ? host_pool() : nullptr;
    if (!pool) {
        for (const CopyJob& j : jobs) memcpy(j.dst, j.src, j.len);
        return;
    }
    std::vector<CopyJob> pieces;
    pieces.reserve(total / kPiece + jobs.size());
    for (const CopyJob& j : jobs)
        for (size_t o = 0; o < j.len; o += kPiece) pieces.push_back({j.dst + o, j.src + o, std::min(kPiece, j.len - o)});
    const std::function<int(int)> one = [&](int i) {
        memcpy(pieces[size_t(i)].dst, pieces[size_t(i)].src, pieces[size_t(i)].len);
        return 0;
    };
    pool->parallel_for(int(pieces.size()), one);
}

// The turn both host pipelines take on the ring: the copy-backs of the piece a slot carries wait in `pending` until the
// slot's event fires; finish(si) then runs them and frees the slot for its next piece.
struct SlotTurns {
    StagingRing& ring;
    std::vector<std::vector<CopyJob>> pending;
    explicit SlotTurns(StagingRing& r) : ring(r), pending(r.slots.size()) {}
    int finish(size_t si) {
        StagingSlot& s = ring.slots[si];
        if (!s.busy) return SWEC_OK;
        SWEC_CUDA(cudaEventSynchronize(s.done));
        parallel_copy(pending[si]);
        pending[si].clear();
        s.busy = false;
        return SWEC_OK;
    }
};

// p[0..n) equally spaced (the k+m slices of ONE allocation, e.g. swec_alloc_pinned_for_device carved up by the caller)?
bool constant_pitch(const uint8_t* const* p, int n, size_t min_pitch, size_t* pitch) {
    if (n < 2) return false;
    if (p[1] <= p[0]) return false;
    const size_t d = size_t(p[1] - p[0]);
    if (d < min_pitch) return false;
    if (d > size_t(0x7fffffff)) return false;  // cudaMemcpy2D pitches are limited (cudaDevAttrMaxPitch): huge shards go one by one
    for (int i = 2; i < n; i++)
        if (p[i] != p[0] + size_t(i) * d) return false;
    *pitch = d;
    return true;
}

}  // namespace

// check = nullptr: out[r] receive the results.  check != nullptr: out[r] are read and compared
// with the computed rows; *check receives the number of mismatching 16-byte vectors.
static int apply_host(swec_encoder_impl* e, const Matrix& rows, const uint8_t* const* in, uint8_t* const* out,
                      size_t n, unsigned long long* check) {
    const int K = rows.cols, R = rows.rows;
    if (R == 0 || n == 0) return SWEC_OK;
    std::lock_guard<std::mutex> lock(e->mu);
    int rc = e->ensure_device();
    if (rc) return rc;

    std::vector<char> in_direct(static_cast<size_t>(K), 0), out_direct(static_cast<size_t>(R), 0);
    const uint8_t* gin[SWEC_MAX_INPUTS];
    uint8_t* gout[SWEC_MAX_SHARDS];
    int ndev = 0, nreach = 0;
    uintptr_t align = 0;
    for (int i = 0; i < K; i++) {
        bool dev;
        const void* g = nullptr;
        in_direct[size_t(i)] = is_pinned_or_device(in[i], &dev, &g);
        gin[i] = static_cast<const uint8_t*>(g);
        ndev += dev;
        nreach += g != nullptr;
        align |= reinterpret_cast<uintptr_t>(g);
    }
    for (int r = 0; r < R; r++) {
        bool dev;
        const void* g = nullptr;
        out_direct[size_t(r)] = is_pinned_or_device(out[r], &dev, &g);
        gout[r] = static_cast<uint8_t*>(const_cast<void*>(g));
        ndev += dev;
        nreach += g != nullptr;
        align |= reinterpret_cast<uintptr_t>(g);
    }
    if (ndev == K + R && !check) {  // everything already lives in HBM
        rc = e->apply(rows, in, out, n, Layout{}, e->stream);
        if (rc) return rc;
        SWEC_CUDA(cudaStreamSynchronize(e->stream));
        return SWEC_OK;
    }
    const long zc_mode = g_opt_host_zero_copy.load();
    const bool zero_copy = !check && (zc_mode == 1 || (zc_mode == 2 && n <= size_t(g_opt_host_zero_copy_max.load())));
    if (zero_copy && nreach == K + R && (align & 15) == 0) {
        // every buffer is mapped pinned (or device) memory: ONE launch reads the data shards over PCIe and writes
        // the parity back; what a 256 KiB-per-shard Encode call costs is this launch and one stream synchronise
        rc = e->apply(rows, gin, gout, n, Layout{}, e->stream);
        if (rc) return rc;
        SWEC_CUDA(cudaStreamSynchronize(e->stream));
        return SWEC_OK;
    }

    // piece size: the call is cut into >= host_pieces pieces (>= host_min_chunk, <= stage_chunk each) travelling on
    // the ring's slots, so that copies in, kernel and copies out of neighbouring pieces overlap inside this one call
    const size_t max_chunk = size_t(std::max(4096l, g_opt_stage_chunk.load()));
    const size_t min_chunk = std::min(max_chunk, size_t(std::max(4096l, g_opt_host_min_chunk.load())));
    const size_t pieces = size_t(std::max(1l, g_opt_host_pieces.load()));
    size_t chunk = (((n + pieces - 1) / pieces) + 4095) & ~size_t(4095);
    chunk = std::min(max_chunk, std::max(min_chunk, chunk));
    chunk = std::min(chunk, (n + 255) & ~size_t(255));
    rc = e->ensure_slots(chunk);
    if (rc) return rc;
    const size_t stride = e->slot_chunk();  // per-stream pitch inside a slot (>= chunk)
    StagingRing& ring = e->ring;

    StagingRing::DrainOnExit drain{ring};
    DeviceCounter counter;
    if (check) {
        SWEC_CUDA(cudaMalloc(reinterpret_cast<void**>(&counter.p), 8));
        SWEC_CUDA(cudaMemset(counter.p, 0, 8));
    }
    unsigned long long* const dev_bad = counter.p;

    SlotTurns turns(ring);

    bool all_in_bounced = true, all_out_bounced = !check, all_in_direct = true, all_out_direct = !check;
    for (int i = 0; i < K; i++) {
        all_in_bounced = all_in_bounced && !in_direct[size_t(i)];
        all_in_direct = all_in_direct && in_direct[size_t(i)];
    }
    for (int r = 0; r < R; r++) {
        all_out_bounced = all_out_bounced && !out_direct[size_t(r)];
        all_out_direct = all_out_direct && out_direct[size_t(r)];
    }
    // pinned callers whose k+m buffers are slices of one allocation: ONE strided DMA each way instead of k + m
    size_t in_pitch = 0, out_pitch = 0;
    const bool in_2d = all_in_direct && constant_pitch(in, K, n, &in_pitch);
    const bool out_2d = all_out_direct && R > 1 && constant_pitch(out, R, n, &out_pitch);
    const bool packed = all_in_bounced && all_out_bounced;

    std::vector<CopyJob> bounce;
    size_t ci = 0;
    for (size_t off = 0; off < n; off += chunk, ci++) {
        const size_t si = ci % ring.slots.size();
        StagingSlot& s = ring.slots[si];
        if ((rc = turns.finish(si))) break;
        const size_t len = std::min(chunk, n - off);
        // Pageable callers (Go heap memory) bounce through the slot anyway, so pack the streams at a
        // pitch that fits this piece: one DMA in, one DMA out instead of k + m small ones.
        const size_t pitch = packed ? ((len + 255) & ~size_t(255)) : stride;
        const uint8_t* din[SWEC_MAX_INPUTS];
        uint8_t* dout[SWEC_MAX_SHARDS];
        bounce.clear();
        for (int i = 0; i < K; i++) {
            din[i] = s.dev + size_t(i) * pitch;
            if (!in_direct[size_t(i)]) bounce.push_back({s.host + size_t(i) * pitch, in[i] + off, len});
        }
        parallel_copy(bounce);
        if (packed && zero_copy && s.host_dev) {
            // pageable caller, short call: the kernel works on the mapped ring itself (reads and writes cross PCIe
            // inside the kernel), so a piece costs one launch instead of H2D + launch + D2H
            for (int i = 0; i < K; i++) din[i] = s.host_dev + size_t(i) * pitch;
            for (int r = 0; r < R; r++) dout[r] = s.host_dev + size_t(K + r) * pitch;
            if ((rc = e->apply(rows, din, dout, len, Layout{}, s.stream))) break;
            for (int r = 0; r < R; r++) turns.pending[si].push_back({out[r] + off, s.host + size_t(K + r) * pitch, len});
            SWEC_CUDA(cudaEventRecord(s.done, s.stream));
            s.busy = true;
            continue;
        }
        if (packed) {
            SWEC_CUDA(cudaMemcpyAsync(s.dev, s.host, size_t(K - 1) * pitch + len, cudaMemcpyHostToDevice, s.stream));
        } else if (in_2d) {
            SWEC_CUDA(cudaMemcpy2DAsync(s.dev, pitch, in[0] + off, in_pitch, len, size_t(K), cudaMemcpyDefault, s.stream));
        } else {
            for (int i = 0; i < K; i++) {
                const uint8_t* src = in_direct[size_t(i)] ? in[i] + off : s.host + size_t(i) * pitch;
                SWEC_CUDA(cudaMemcpyAsync(s.dev + size_t(i) * pitch, src, len, cudaMemcpyDefault, s.stream));
            }
        }
        for (int r = 0; r < R; r++) dout[r] = s.dev + size_t(K + r) * pitch;
        if ((rc = e->apply(rows, din, dout, len, Layout{}, s.stream))) break;
        if (packed) {
            SWEC_CUDA(cudaMemcpyAsync(s.host + size_t(K) * pitch, dout[0], size_t(R - 1) * pitch + len,
                                      cudaMemcpyDeviceToHost, s.stream));
            for (int r = 0; r < R; r++) turns.pending[si].push_back({out[r] + off, s.host + size_t(K + r) * pitch, len});
        } else if (out_2d) {
            SWEC_CUDA(cudaMemcpy2DAsync(out[0] + off, out_pitch, dout[0], pitch, len, size_t(R), cudaMemcpyDefault, s.stream));
        } else {
            if (check) {  // bring the caller's copy of every row next to the computed one and compare in HBM
                bounce.clear();
                for (int r = 0; r < R; r++)
                    if (!out_direct[size_t(r)]) bounce.push_back({s.host + size_t(K + r) * stride, out[r] + off, len});
                parallel_copy(bounce);
            }
            for (int r = 0; r < R; r++) {
                if (check) {
                    uint8_t* theirs = s.dev + size_t(K + R + r) * stride;
                    const uint8_t* src = out_direct[size_t(r)] ? out[r] + off : s.host + size_t(K + r) * stride;
                    SWEC_CUDA(cudaMemcpyAsync(theirs, src, len, cudaMemcpyDefault, s.stream));
                    SWEC_CUDA(launch_compare(dout[r], theirs, len, dev_bad, s.stream));
                } else if (out_direct[size_t(r)]) {
                    SWEC_CUDA(cudaMemcpyAsync(out[r] + off, dout[r], len, cudaMemcpyDefault, s.stream));
                } else {
                    uint8_t* back = s.host + size_t(K + r) * stride;
                    SWEC_CUDA(cudaMemcpyAsync(back, dout[r], len, cudaMemcpyDeviceToHost, s.stream));
                    turns.pending[si].push_back({out[r] + off, back, len});
                }
            }
        }
        SWEC_CUDA(cudaEventRecord(s.done, s.stream));
        s.busy = true;
    }
    for (size_t i = 0; i < ring.slots.size(); i++) {
        // drain in submission order so that copy-backs of early pieces overlap the GPU work of late ones
        const int rc2 = turns.finish((ci + i) % ring.slots.size());
        if (!rc) rc = rc2;
    }
    if (check && !rc && cudaMemcpy(check, dev_bad, 8, cudaMemcpyDeviceToHost) != cudaSuccess)
        rc = cuda_fail(cudaGetLastError(), "reading the mismatch counter");
    return rc;
}

// Largest interval the packed path takes (bigger ones stream through apply_host): small on purpose — the
// ring behind it is 3 slots x (k+2m) streams x this, and needle-sized intervals gain nothing from more.
static size_t packed_max_bytes() {
    return std::min(size_t(std::max(4096l, g_opt_stage_chunk.load())), size_t(2) << 20);
}

// Many small intervals that share one matrix (degraded reads behind one dead server): pack them
// back to back (each padded to 16 bytes) into slot-sized launches so the per-call costs — stream
// round trip, launch, DMA set-up — are paid once per ~chunk instead of once per needle.
struct Segment {
    std::vector<const uint8_t*> in;  // K pointers
    std::vector<uint8_t*> out;       // R pointers
    size_t len;
};

static int apply_host_packed(swec_encoder_impl* e, const Matrix& rows, const std::vector<Segment>& segs) {
    const int K = rows.cols, R = rows.rows;
    if (R == 0 || segs.empty()) return SWEC_OK;
    std::lock_guard<std::mutex> lock(e->mu);
    int rc = e->ensure_device();
    if (rc) return rc;
    // size the ring for THIS batch (a lone degraded read must not pin 3 x 18 x 16 MiB): everything packed
    // back to back, capped by the configured chunk; ensure_slots only ever grows an existing ring
    const size_t max_chunk = packed_max_bytes();
    size_t packed = 0;
    for (const Segment& sg : segs) packed += (sg.len + 15) & ~size_t(15);
    const size_t chunk = std::min(max_chunk, (packed + 65535) & ~size_t(65535));
    if ((rc = e->ensure_slots(chunk))) return rc;
    const size_t stride = e->slot_chunk();
    StagingRing& ring = e->ring;
    StagingRing::DrainOnExit drain{ring};
    SlotTurns turns(ring);
    size_t si = 0, fill = 0, nflush = 0;
    auto flush = [&]() -> int {
        if (fill == 0) return SWEC_OK;
        StagingSlot& sl = ring.slots[si];
        const uint8_t* din[SWEC_MAX_INPUTS];
        uint8_t* dout[SWEC_MAX_SHARDS];
        const long zc_mode = g_opt_host_zero_copy.load();
        // zero-copy pays for one needle per call and costs when many needles fill slot after slot (earlier GPU
        // generation; scripts/bench_needles.py measures it) — full slots keep the strided-DMA pipeline
        const size_t packed_zero_copy_max = std::min(size_t(g_opt_host_zero_copy_max.load()), size_t(256) << 10);
        if (sl.host_dev && (zc_mode == 1 || (zc_mode == 2 && fill <= packed_zero_copy_max))) {
            // needle-sized batches: the kernel works on the mapped ring itself — one launch instead of
            // strided DMA in + launch + strided DMA out (what a degraded read waits for is API round trips)
            for (int i = 0; i < K; i++) din[i] = sl.host_dev + size_t(i) * stride;
            for (int r = 0; r < R; r++) dout[r] = sl.host_dev + size_t(K + r) * stride;
            const int rc2 = e->apply(rows, din, dout, fill, Layout{}, sl.stream);
            if (rc2) return rc2;
        } else {
            for (int i = 0; i < K; i++) din[i] = sl.dev + size_t(i) * stride;
            // the K input streams sit at pitch `stride` in both buffers: one strided DMA instead of K small ones
            SWEC_CUDA(cudaMemcpy2DAsync(sl.dev, stride, sl.host, stride, fill, size_t(K), cudaMemcpyHostToDevice, sl.stream));
            for (int r = 0; r < R; r++) dout[r] = sl.dev + size_t(K + r) * stride;
            const int rc2 = e->apply(rows, din, dout, fill, Layout{}, sl.stream);
            if (rc2) return rc2;
            SWEC_CUDA(cudaMemcpy2DAsync(sl.host + size_t(K) * stride, stride, dout[0], stride, fill, size_t(R),
                                        cudaMemcpyDeviceToHost, sl.stream));
        }
        SWEC_CUDA(cudaEventRecord(sl.done, sl.stream));
        sl.busy = true;
        fill = 0;
        si = (++nflush) % ring.slots.size();
        return turns.finish(si);  // the slot we are about to fill must be drained
    };
    for (const Segment& sg : segs) {
        const size_t padded = (sg.len + 15) & ~size_t(15);
        if (padded > stride) {  // larger than a slot: not a "small interval" — caller should not batch it
            return fail(SWEC_ERR_INVALID_ARG, "batched interval larger than the staging chunk");
        }
        if (fill + padded > stride && (rc = flush())) return rc;
        StagingSlot& sl = ring.slots[si];
        for (int i = 0; i < K; i++) {
            uint8_t* dst = sl.host + size_t(i) * stride + fill;
            memcpy(dst, sg.in[i], sg.len);
            if (padded > sg.len) memset(dst + sg.len, 0, padded - sg.len);
        }
        for (int r = 0; r < R; r++) turns.pending[si].push_back({sg.out[r], sl.host + size_t(K + r) * stride + fill, sg.len});
        fill += padded;
    }
    if ((rc = flush())) return rc;
    for (size_t i = 0; i < ring.slots.size(); i++)
        if ((rc = turns.finish(i))) return rc;
    return SWEC_OK;
}

Matrix parity_rows(const swec_encoder_impl* e) {
    Matrix rows(e->m, e->k);
    memcpy(rows.v.data(), e->gen.row(e->k), rows.v.size());
    return rows;
}

// What a reconstruct call rebuilds, decided once from the presence mask: the fused matrix, the shards it reads and the
// shards it writes (none when every shard is present, or when only parity is missing and data_only is set).
struct ReconstructPlan {
    bool all_present = false;
    std::vector<int> ins, outs;
    Matrix fused;

    // the caller's buffers of the plan's inputs and outputs; every shard to rebuild needs one
    int gather(uint8_t* const* shards, const uint8_t** in, uint8_t** out) const {
        for (size_t i = 0; i < ins.size(); i++) in[i] = shards[ins[i]];
        for (size_t i = 0; i < outs.size(); i++) {
            out[i] = shards[outs[i]];
            if (!out[i]) return fail(SWEC_ERR_INVALID_ARG, "missing shard has no buffer");
        }
        return SWEC_OK;
    }
};

static int plan_reconstruct(const swec_encoder_impl* e, const uint8_t* present, int data_only, ReconstructPlan* p) {
    int npresent = 0;
    for (int i = 0; i < e->k + e->m; i++) npresent += present[i] ? 1 : 0;
    p->all_present = npresent == e->k + e->m;
    if (p->all_present) return SWEC_OK;
    if (npresent < e->k || !rs_reconstruct_plan(e->gen, e->k, present, data_only != 0, &p->ins, &p->outs, &p->fused))
        return fail(SWEC_ERR_TOO_FEW_SHARDS, "fewer than data_shards shards present");
    return SWEC_OK;
}

}  // namespace swec

// =================================================================== C ABI

using namespace swec;

extern "C" {

const char* swec_version(void) { return "swec 0.1 (sm_90a)"; }

const char* swec_strerror(int status) {
    switch (status) {
        case SWEC_OK: return "ok";
        case SWEC_ERR_INVALID_ARG: return "invalid argument";
        case SWEC_ERR_TOO_FEW_SHARDS: return "too few shards given";
        case SWEC_ERR_CUDA: return "CUDA error";
        case SWEC_ERR_IO: return "I/O error";
        case SWEC_ERR_NOMEM: return "out of memory";
        case SWEC_ERR_SHARD_SIZE: return "shard sizes do not match";
        case SWEC_ERR_NO_DEVICE: return "no usable CUDA device (there is no CPU fallback)";
        case SWEC_ERR_JIT: return "run-time kernel specialisation failed";
        case SWEC_ERR_NO_LIVE_NEEDLES: return "ec volume has no live entries";
        case SWEC_ERR_NOT_FOUND: return "needle not found";
        case SWEC_ERR_DELETED: return "needle already deleted";
        default: return "unknown error";
    }
}

const char* swec_last_error(void) { return last_error(); }

int swec_device_count(int* count) {
    int n = 0;
    const cudaError_t e = cudaGetDeviceCount(&n);
    if (count) *count = e == cudaSuccess ? n : 0;
    if (e != cudaSuccess) {  // whatever the driver's reason, the caller's answer is the same: no device
        cudaGetLastError();
        cuda_fail(e, "cudaGetDeviceCount");  // records the detail text
        return SWEC_ERR_NO_DEVICE;
    }
    return n > 0 ? SWEC_OK : fail(SWEC_ERR_NO_DEVICE, "no CUDA devices");
}

// Placement order for a process (or a launcher) that drives several GPUs: device ids interleaved over the host's
// NUMA nodes — 0,4,1,5,2,6,3,7 on a box with GPUs 0-3 on socket 0 and 4-7 on socket 1.  Host-fed work is bound by
// what ONE socket can DMA (scripts/pcie_socket_probe.py measures it), so the first n devices of this
// order spread n concurrent volumes over both sockets' memory controllers and root complexes instead of filling
// socket 0 first.  Devices whose node is unknown keep their index order at the end.
int swec_device_spread_order(int* order, int capacity, int* count) {
    if (!order || !count || capacity <= 0) return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    int n = 0;
    const cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        cudaGetLastError();
        *count = 0;
        return fail(SWEC_ERR_NO_DEVICE, "no CUDA devices");
    }
    std::map<int, std::vector<int>> by_node;  // node → devices, both ascending
    for (int d = 0; d < n; d++) by_node[device_numa_node(d)].push_back(d);
    std::vector<int> out;
    for (size_t round = 0; out.size() < size_t(n); round++)
        for (auto& kv : by_node)
            if (round < kv.second.size()) out.push_back(kv.second[round]);
    *count = std::min(n, capacity);
    for (int i = 0; i < *count; i++) order[i] = out[size_t(i)];
    return SWEC_OK;
}

uint64_t swec_kernel_launches(void) { return g_kernel_launches.load(); }

void swec_shutdown(void) {
    jit_shutdown();
    file_pipeline_trim();
}

int swec_jit_stats(uint64_t* nvrtc_compiles, uint64_t* disk_cache_hits, int* aot_matrices, uint64_t* aot_launches) {
    if (aot_launches) *aot_launches = aot_recon_launches();
    if (nvrtc_compiles) *nvrtc_compiles = jit_compile_count();
    if (disk_cache_hits) *disk_cache_hits = jit_disk_hit_count();
    if (aot_matrices) *aot_matrices = aot_recon_count();
    return SWEC_OK;
}

int swec_debug_power_state(int device, double* heat_ms, int* low_power) {
    if (device >= 0) SWEC_CUDA(cudaSetDevice(device));
    if (heat_ms) *heat_ms = power_heat_ms();
    if (low_power) *low_power = low_power_now() ? 1 : 0;
    return SWEC_OK;
}

int swec_debug_jit_compile(int r, int k, const uint8_t* rows, size_t* cubin_bytes, int* xtime_steps, int* xor_ops) {
    if (r <= 0 || k <= 0 || k > SWEC_MAX_INPUTS || !rows) return fail(SWEC_ERR_INVALID_ARG, "bad matrix");
    Matrix m(r, k);
    memcpy(m.v.data(), rows, m.v.size());
    return jit_debug_compile(m, cubin_bytes, xtime_steps, xor_ops);
}

int swec_set_option(const char* name, long value) {
    if (!name) return fail(SWEC_ERR_INVALID_ARG, "NULL option name");
    const std::string n(name);
    if (n == "enc_threads" && (value == 128 || value == 256 || value == 512)) g_opt_enc_threads = value;
    else if (n == "enc_unroll" && (value == 1 || value == 2)) g_opt_enc_unroll = value;
    else if (n == "ctas_per_sm" && value >= 0 && value <= 64) g_opt_ctas_per_sm = value;
    else if (n == "stage_chunk" && value >= 4096) g_opt_stage_chunk = (value + 255) & ~255l;
    else if (n == "stage_slots" && value >= 2 && value <= 16) g_opt_stage_slots = value;
    else if (n == "host_pieces" && value >= 1 && value <= 64) g_opt_host_pieces = value;
    else if (n == "host_min_chunk" && value >= 4096) g_opt_host_min_chunk = (value + 4095) & ~4095l;
    else if (n == "file_direct_io" && value >= 0 && value <= 3) g_opt_file_direct_io = value;
    else if (n == "host_zero_copy" && value >= 0 && value <= 2) g_opt_host_zero_copy = value;
    else if (n == "host_zero_copy_max" && value >= 0) g_opt_host_zero_copy_max = value;
    else if (n == "jit_min_bytes" && value >= 0) g_opt_jit_min_bytes = value;
    else if (n == "jit" && (value == 0 || value == 1)) g_opt_jit_enabled = value;
    else if (n == "xt_variant" && value >= 0 && value <= 3) g_opt_xt_variant = value;
    else if (n == "use_aot" && (value == 0 || value == 1)) g_opt_use_aot = value;
    else if (n == "jit_share_powers" && (value == 0 || value == 1)) g_opt_jit_share_powers = value;
    else if (n == "power_mode" && value >= 0 && value <= 2) g_opt_power_mode = value;
    else return fail(SWEC_ERR_INVALID_ARG, "unknown option or value out of range: " + n);
    return SWEC_OK;
}

int swec_encoder_new(int k, int m, int device, swec_encoder** out) {
    if (!out) return fail(SWEC_ERR_INVALID_ARG, "out is NULL");
    *out = nullptr;
    // reedsolomon.New: ErrInvShardNum for non-positive counts; SeaweedFS caps the total at
    // MaxShardCount (ec_encoder.go:23,81)
    if (k <= 0 || m <= 0 || k + m > SWEC_MAX_SHARDS)
        return fail(SWEC_ERR_INVALID_ARG, "need data_shards > 0, parity_shards > 0, total <= 32");
    swec_encoder* e = new (std::nothrow) swec_encoder();
    if (!e) return fail(SWEC_ERR_NOMEM, "out of memory");
    e->k = k;
    e->m = m;
    e->device = device;
    e->gen = rs_generator(k, m);
    e->rs10x4 = (k == 10 && m == 4);
    *out = e;
    return SWEC_OK;
}

void swec_encoder_free(swec_encoder* e) { delete e; }

int swec_encoder_matrix(const swec_encoder* e, uint8_t* out) {
    if (!e || !out) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    memcpy(out, e->gen.v.data(), e->gen.v.size());
    return SWEC_OK;
}

int swec_reconstruct_matrix(const swec_encoder* e, const uint8_t* present, int data_only, int* inputs,
                            int* outputs, int* n_outputs, uint8_t* rows) {
    if (!e || !present || !inputs || !outputs || !n_outputs || !rows) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    std::vector<int> in, outv;
    Matrix fused;
    if (!rs_reconstruct_plan(e->gen, e->k, present, data_only != 0, &in, &outv, &fused))
        return fail(SWEC_ERR_TOO_FEW_SHARDS, "fewer than data_shards shards present");
    for (int i = 0; i < e->k; i++) inputs[i] = in[size_t(i)];
    *n_outputs = int(outv.size());
    for (size_t i = 0; i < outv.size(); i++) outputs[i] = outv[i];
    if (!fused.v.empty()) memcpy(rows, fused.v.data(), fused.v.size());
    return SWEC_OK;
}

int swec_encode(swec_encoder* e, uint8_t* const* shards, size_t n) {
    if (!e || !shards) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    if (n == 0) return fail(SWEC_ERR_INVALID_ARG, "shard_len is 0 (ErrShardNoData)");
    for (int i = 0; i < e->k + e->m; i++)
        if (!shards[i]) return fail(SWEC_ERR_INVALID_ARG, "NULL shard");
    return apply_host(e, parity_rows(e), shards, shards + e->k, n, nullptr);
}

int swec_reconstruct(swec_encoder* e, uint8_t* const* shards, const uint8_t* present, size_t n, int data_only) {
    if (!e || !shards || !present) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    ReconstructPlan p;
    int rc = plan_reconstruct(e, present, data_only, &p);
    if (rc || p.all_present) return rc;
    if (n == 0) return fail(SWEC_ERR_INVALID_ARG, "shard_len is 0 (ErrShardNoData)");
    if (p.outs.empty()) return SWEC_OK;
    const uint8_t* ins[SWEC_MAX_SHARDS];
    uint8_t* outs[SWEC_MAX_SHARDS];
    if ((rc = p.gather(shards, ins, outs))) return rc;
    return apply_host(e, p.fused, ins, outs, n, nullptr);
}

int swec_reconstruct_batch(swec_encoder* e, const swec_reconstruct_item* items, int n_items) {
    if (!e || (n_items > 0 && !items)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    const int total = e->k + e->m;
    const size_t chunk = swec::packed_max_bytes();
    // group by (presence mask, data_only); big items take the ordinary streaming path
    struct Group {
        ReconstructPlan plan;
        std::vector<Segment> segs;
    };
    std::map<std::vector<uint8_t>, Group> groups;
    for (int it = 0; it < n_items; it++) {
        const swec_reconstruct_item& item = items[it];
        if (!item.shards || !item.present) return fail(SWEC_ERR_INVALID_ARG, "NULL item field");
        std::vector<uint8_t> key(item.present, item.present + total);
        for (auto& b : key) b = b ? 1 : 0;
        key.push_back(item.data_only ? 1 : 0);
        auto found = groups.find(key);
        if (found == groups.end()) {
            Group g;
            if (const int rc = plan_reconstruct(e, key.data(), item.data_only, &g.plan)) return rc;
            found = groups.emplace(key, std::move(g)).first;
        }
        Group& g = found->second;
        if (g.plan.all_present) continue;
        if (item.shard_len == 0) return fail(SWEC_ERR_INVALID_ARG, "shard_len is 0 (ErrShardNoData)");
        if (((item.shard_len + 15) & ~size_t(15)) > chunk) {
            const int rc = swec_reconstruct(e, item.shards, item.present, item.shard_len, item.data_only);
            if (rc) return rc;
            continue;
        }
        if (g.plan.outs.empty()) continue;
        Segment sg{std::vector<const uint8_t*>(g.plan.ins.size()), std::vector<uint8_t*>(g.plan.outs.size()), item.shard_len};
        if (const int rc = g.plan.gather(item.shards, sg.in.data(), sg.out.data())) return rc;
        g.segs.push_back(std::move(sg));
    }
    for (auto& kv : groups)
        if (const int rc = apply_host_packed(e, kv.second.plan.fused, kv.second.segs)) return rc;
    return SWEC_OK;
}

// ---- one call, several GPUs: column ranges are independent (parity_p[x] depends only on data_*[x]),
// so a host-buffer call can be cut into contiguous byte ranges, one per encoder handle (= per GPU), each
// range travelling over its own GPU's PCIe link through that handle's staging ring.  No collective.

}  // extern "C"

namespace {

// THE split rule (swec_encode_multi, swec_reconstruct_multi, swec_alloc_pinned_shards agree on it): range g of n
// bytes over n_encs handles starts at begin[g]; 4 KiB granularity keeps every range page- and 16-byte aligned
// relative to the caller's buffers
std::vector<size_t> column_split(int n_encs, size_t n) {
    const size_t gran = 4096;
    const size_t units = (n + gran - 1) / gran;
    std::vector<size_t> begin(size_t(n_encs) + 1, 0);
    for (int g = 0; g <= n_encs; g++) begin[size_t(g)] = std::min(n, units * size_t(g) / size_t(n_encs) * gran);
    begin[size_t(n_encs)] = n;
    return begin;
}

template <class Fn>  // fn(g, offset, len) → status, run concurrently for every non-empty range
int split_columns(int n_encs, size_t n, Fn&& fn) {
    const std::vector<size_t> begin = column_split(n_encs, n);
    std::vector<int> rc(size_t(n_encs), SWEC_OK);
    std::vector<std::string> msg(static_cast<size_t>(n_encs));
    std::vector<std::thread> threads;
    for (int g = 0; g < n_encs; g++) {
        const size_t off = begin[size_t(g)], len = begin[size_t(g) + 1] - off;
        if (!len) continue;
        threads.emplace_back([&, g, off, len] {
            rc[size_t(g)] = fn(g, off, len);
            if (rc[size_t(g)]) msg[size_t(g)] = last_error();  // thread-local: carry it to the caller's thread
        });
    }
    for (auto& t : threads) t.join();
    for (int g = 0; g < n_encs; g++)
        if (rc[size_t(g)]) return fail(rc[size_t(g)], msg[size_t(g)]);
    return SWEC_OK;
}

int check_group(swec_encoder* const* encs, int n_encs) {
    if (!encs || n_encs <= 0 || n_encs > 64) return fail(SWEC_ERR_INVALID_ARG, "need 1..64 encoder handles");
    for (int g = 0; g < n_encs; g++) {
        if (!encs[g]) return fail(SWEC_ERR_INVALID_ARG, "NULL encoder handle");
        if (encs[g]->k != encs[0]->k || encs[g]->m != encs[0]->m)
            return fail(SWEC_ERR_INVALID_ARG, "encoder handles of one group must share the EC ratio");
        for (int h = 0; h < g; h++)
            if (encs[h] == encs[g]) return fail(SWEC_ERR_INVALID_ARG, "the same encoder handle appears twice (its staging ring serialises)");
    }
    return SWEC_OK;
}

}  // namespace

extern "C" {

int swec_encode_multi(swec_encoder* const* encs, int n_encs, uint8_t* const* shards, size_t n) {
    int rc = check_group(encs, n_encs);
    if (rc) return rc;
    if (!shards) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    if (n == 0) return fail(SWEC_ERR_INVALID_ARG, "shard_len is 0 (ErrShardNoData)");
    const int total = encs[0]->k + encs[0]->m;
    for (int i = 0; i < total; i++)
        if (!shards[i]) return fail(SWEC_ERR_INVALID_ARG, "NULL shard");
    return split_columns(n_encs, n, [&](int g, size_t off, size_t len) {
        uint8_t* sub[SWEC_MAX_SHARDS];
        for (int i = 0; i < total; i++) sub[i] = shards[i] + off;
        return swec_encode(encs[g], sub, len);
    });
}

// Host buffers laid out for a column-split call: byte range g of every shard lives on the NUMA node of the GPU that
// will DMA it.  A plain pinned buffer sits on one socket, and the GPUs of the other socket then pull their ranges
// across the inter-socket link (scripts/bench_group.py --numa-split measures the difference).
int swec_alloc_pinned_shards(swec_encoder* const* encs, int n_encs, int n_shards, size_t shard_len, uint8_t** shards) {
    int rc = check_group(encs, n_encs);
    if (rc) return rc;
    if (!shards || n_shards <= 0 || n_shards > SWEC_MAX_SHARDS || shard_len == 0) return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    const size_t pitch = (shard_len + 4095) & ~size_t(4095);
    const size_t total = pitch * size_t(n_shards);
    void* base = mmap(nullptr, total, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (base == MAP_FAILED) return fail(SWEC_ERR_NOMEM, "mmap of the shard buffers failed");
    const std::vector<size_t> begin = column_split(n_encs, shard_len);
    for (int g = 0; g < n_encs; g++) {
        const int node = device_numa_node(encs[g]->device);
        // the end of the last range is rounded up to the page so that the tail page has a home too
        const size_t lo = begin[size_t(g)], hi = g + 1 == n_encs ? pitch : begin[size_t(g) + 1];
        for (int i = 0; i < n_shards && hi > lo; i++) bind_to_node(static_cast<uint8_t*>(base) + size_t(i) * pitch + lo, hi - lo, node);
    }
    const cudaError_t e = register_mapped(base, total);
    if (e != cudaSuccess) {
        munmap(base, total);
        return cuda_fail(e, "cudaHostRegister of the shard buffers");
    }
    for (int i = 0; i < n_shards; i++) shards[i] = static_cast<uint8_t*>(base) + size_t(i) * pitch;
    return SWEC_OK;
}

int swec_reconstruct_multi(swec_encoder* const* encs, int n_encs, uint8_t* const* shards, const uint8_t* present,
                           size_t n, int data_only) {
    int rc = check_group(encs, n_encs);
    if (rc) return rc;
    if (!shards || !present) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    const int total = encs[0]->k + encs[0]->m;
    ReconstructPlan p;
    if ((rc = plan_reconstruct(encs[0], present, data_only, &p)) || p.all_present) return rc;
    if (n == 0) return fail(SWEC_ERR_INVALID_ARG, "shard_len is 0 (ErrShardNoData)");
    const uint8_t* ins[SWEC_MAX_SHARDS];
    uint8_t* outs[SWEC_MAX_SHARDS];
    if ((rc = p.gather(shards, ins, outs))) return rc;
    return split_columns(n_encs, n, [&](int g, size_t off, size_t len) {
        uint8_t* sub[SWEC_MAX_SHARDS];
        for (int i = 0; i < total; i++) sub[i] = shards[i] ? shards[i] + off : nullptr;
        return swec_reconstruct(encs[g], sub, present, len, data_only);
    });
}

int swec_verify(swec_encoder* e, uint8_t* const* shards, size_t n, int* ok) {
    if (!e || !shards || !ok) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    if (n == 0) return fail(SWEC_ERR_INVALID_ARG, "shard_len is 0");
    unsigned long long bad = 0;
    const int rc = apply_host(e, parity_rows(e), shards, shards + e->k, n, &bad);
    *ok = rc == SWEC_OK && bad == 0;
    return rc;
}

// ---- device-resident

// `stream` is a plain cudaStream_t; NULL is CUDA's default stream, exactly as in the runtime API
static cudaStream_t pick_stream(swec_encoder*, void* stream) { return static_cast<cudaStream_t>(stream); }

int swec_encode_device(swec_encoder* e, const void* const* data, void* const* parity, size_t n, void* stream) {
    if (!e || !data || !parity) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    std::lock_guard<std::mutex> lock(e->mu);
    int rc = e->ensure_device();
    if (rc) return rc;
    return e->apply(parity_rows(e), reinterpret_cast<const uint8_t* const*>(data),
                    reinterpret_cast<uint8_t* const*>(parity), n, Layout{}, pick_stream(e, stream));
}

int swec_reconstruct_device(swec_encoder* e, void* const* shards, const uint8_t* present, size_t n, int data_only,
                            void* stream) {
    if (!e || !shards || !present) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    ReconstructPlan p;
    int rc = plan_reconstruct(e, present, data_only, &p);
    if (rc || p.outs.empty()) return rc;
    const uint8_t* ins[SWEC_MAX_SHARDS];
    uint8_t* outs[SWEC_MAX_SHARDS];
    if ((rc = p.gather(reinterpret_cast<uint8_t* const*>(shards), ins, outs))) return rc;
    std::lock_guard<std::mutex> lock(e->mu);
    if ((rc = e->ensure_device())) return rc;
    return e->apply(p.fused, ins, outs, n, Layout{}, pick_stream(e, stream));
}

int swec_apply_device(swec_encoder* e, int r, int k, const uint8_t* rows, const void* const* in, void* const* out,
                      size_t n, void* stream) {
    if (!e || !rows || !in || !out || r <= 0 || k <= 0 || k > SWEC_MAX_INPUTS || r > SWEC_MAX_SHARDS)
        return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    Matrix m(r, k);
    memcpy(m.v.data(), rows, m.v.size());
    std::lock_guard<std::mutex> lock(e->mu);
    int rc = e->ensure_device();
    if (rc) return rc;
    return e->apply(m, reinterpret_cast<const uint8_t* const*>(in), reinterpret_cast<uint8_t* const*>(out), n,
                    Layout{}, pick_stream(e, stream));
}

int swec_encode_volume_device(swec_encoder* e, const void* dat_v, int64_t dat_size, int64_t large, int64_t small,
                              void* const* parity, void* stream) {
    if (!e || !dat_v || !parity || dat_size < 0 || large <= 0 || small <= 0)
        return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    const uint8_t* dat = static_cast<const uint8_t*>(dat_v);
    const int k = e->k, m = e->m;
    std::lock_guard<std::mutex> lock(e->mu);
    int rc = e->ensure_device();
    if (rc) return rc;
    cudaStream_t s = pick_stream(e, stream);
    const Matrix rows = parity_rows(e);
    bool horner = is_rs10x4_parity(*e, rows);
    if (!horner && e->m <= SWEC_MAX_OUTPUTS && g_opt_jit_enabled.load() && jit_available()) {
        std::shared_ptr<JitKernel> jk;
        horner = jit_get(e, rows, &jk) == SWEC_OK;
    }

    // one region = `nrows` rows of k blocks of `block` bytes starting at `base`; parity offset `poff`
    auto region = [&](const uint8_t* base, int64_t block, int64_t nrows, int64_t poff) -> int {
        const uint8_t* ins[SWEC_MAX_SHARDS];
        uint8_t* outs[SWEC_MAX_SHARDS];
        const bool vec_ok = horner && block % 16 == 0 && (reinterpret_cast<uintptr_t>(base) & 15) == 0;
        if (vec_ok || nrows == 1) {
            for (int i = 0; i < k; i++) ins[i] = base + int64_t(i) * block;
            for (int p = 0; p < m; p++) outs[p] = static_cast<uint8_t*>(parity[p]) + poff;
            Layout lay;
            lay.blocked = nrows > 1;
            lay.block_bytes = uint64_t(block);
            return e->apply(rows, ins, outs, size_t(nrows * block), lay, s);
        }
        for (int64_t r = 0; r < nrows; r++) {  // unaligned / table path: one flat launch per row
            for (int i = 0; i < k; i++) ins[i] = base + (r * k + i) * block;
            for (int p = 0; p < m; p++) outs[p] = static_cast<uint8_t*>(parity[p]) + poff + r * block;
            const int rc2 = e->apply(rows, ins, outs, size_t(block), Layout{}, s);
            if (rc2) return rc2;
        }
        return SWEC_OK;
    };

    const StripeGeometry g(dat_size, k, large, small);
    if (g.large_rows && (rc = region(dat, large, g.large_rows, 0))) return rc;
    if (g.small_rows && (rc = region(dat + g.small_dat_offset(), small, g.small_rows, g.small_shard_offset()))) return rc;
    if (g.tail > 0) {  // last row: bytes past EOF read as zero (ec_encoder.go:258-262)
        struct Scratch {  // stream-ordered: freed after the work queued on s, on every exit path
            uint8_t* p = nullptr;
            cudaStream_t s;
            ~Scratch() {
                if (p) cudaFreeAsync(p, s);
            }
        } scratch{nullptr, s};
        SWEC_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&scratch.p), size_t(g.small_row()), s));
        SWEC_CUDA(cudaMemsetAsync(scratch.p, 0, size_t(g.small_row()), s));
        SWEC_CUDA(cudaMemcpyAsync(scratch.p, dat + g.tail_dat_offset(), size_t(g.tail), cudaMemcpyDeviceToDevice, s));
        rc = region(scratch.p, small, 1, g.tail_shard_offset());
        if (rc) return rc;
    }
    return SWEC_OK;
}

int swec_extract_data_shard_device(swec_encoder* e, const void* dat_v, int64_t dat_size, int64_t large, int64_t small,
                                   int shard_id, void* shard_out, void* stream) {
    if (!e || !dat_v || !shard_out || shard_id < 0 || shard_id >= e->k || dat_size < 0 || large <= 0 || small <= 0)
        return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    const uint8_t* dat = static_cast<const uint8_t*>(dat_v);
    uint8_t* dst = static_cast<uint8_t*>(shard_out);
    std::lock_guard<std::mutex> lock(e->mu);
    int rc = e->ensure_device();
    if (rc) return rc;
    cudaStream_t s = pick_stream(e, stream);
    const StripeGeometry g(dat_size, e->k, large, small);
    if (g.large_rows)
        SWEC_CUDA(cudaMemcpy2DAsync(dst, size_t(large), dat + int64_t(shard_id) * large, size_t(g.large_row()), size_t(large),
                                    size_t(g.large_rows), cudaMemcpyDeviceToDevice, s));
    if (g.small_rows)
        SWEC_CUDA(cudaMemcpy2DAsync(dst + g.small_shard_offset(), size_t(small), dat + g.small_dat_offset() + int64_t(shard_id) * small,
                                    size_t(g.small_row()), size_t(small), size_t(g.small_rows), cudaMemcpyDeviceToDevice, s));
    if (g.tail > 0) {
        uint8_t* d3 = dst + g.tail_shard_offset();
        const int64_t have = g.tail_bytes(shard_id);
        if (have) SWEC_CUDA(cudaMemcpyAsync(d3, dat + g.tail_dat_offset() + int64_t(shard_id) * small, size_t(have), cudaMemcpyDeviceToDevice, s));
        if (have < small) SWEC_CUDA(cudaMemsetAsync(d3 + have, 0, size_t(small - have), s));
    }
    return SWEC_OK;
}

int swec_write_dat_device(swec_encoder* e, const void* const* data_shards, int64_t dat_size, int64_t large, int64_t small,
                          void* dat_out, void* stream) {
    if (!e || !data_shards || !dat_out || dat_size < 0 || large <= 0 || small <= 0)
        return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    const int k = e->k;
    for (int i = 0; i < k; i++)
        if (!data_shards[i]) return fail(SWEC_ERR_INVALID_ARG, "NULL data shard");
    uint8_t* dat = static_cast<uint8_t*>(dat_out);
    std::lock_guard<std::mutex> lock(e->mu);
    int rc = e->ensure_device();
    if (rc) return rc;
    cudaStream_t s = pick_stream(e, stream);
    // WriteDatFile's loops (ec_decoder.go:197-219): `for datFileSize >= dataShards*LargeBlockSize` copies large blocks
    // round-robin, then small blocks until the size is used up — the last block short
    const StripeGeometry g(dat_size, k, large, small);
    for (int i = 0; i < k; i++) {
        const uint8_t* sh = static_cast<const uint8_t*>(data_shards[i]);
        if (g.large_rows)
            SWEC_CUDA(cudaMemcpy2DAsync(dat + int64_t(i) * large, size_t(g.large_row()), sh, size_t(large), size_t(large),
                                        size_t(g.large_rows), cudaMemcpyDeviceToDevice, s));
        if (g.small_rows)
            SWEC_CUDA(cudaMemcpy2DAsync(dat + g.small_dat_offset() + int64_t(i) * small, size_t(g.small_row()), sh + g.small_shard_offset(),
                                        size_t(small), size_t(small), size_t(g.small_rows), cudaMemcpyDeviceToDevice, s));
        if (const int64_t have = g.tail_bytes(i))
            SWEC_CUDA(cudaMemcpyAsync(dat + g.tail_dat_offset() + int64_t(i) * small, sh + g.tail_shard_offset(), size_t(have),
                                      cudaMemcpyDeviceToDevice, s));
    }
    return SWEC_OK;
}

int swec_locate_damage_device(swec_encoder* e, const void* const* shards, size_t n, int radius, swec_damage_report* report,
                              swec_damage_range* ranges, int ranges_cap, int* n_ranges, void* stream) {
    if (!e || !shards) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    int rc = check_locate_args(e->m, radius, report, ranges, ranges_cap);
    if (rc) return rc;
    const int k = e->k, m = e->m;
    for (int i = 0; i < k + m; i++)
        if (!shards[i]) return fail(SWEC_ERR_INVALID_ARG, "NULL shard");
    const uint8_t* const* sh = reinterpret_cast<const uint8_t* const*>(shards);
    std::lock_guard<std::mutex> lock(e->mu);
    if ((rc = e->ensure_device())) return rc;
    cudaStream_t s = pick_stream(e, stream);
    const Matrix rows = parity_rows(e);
    DamageLocator locator;
    if ((rc = locator.init(rows, int64_t(n), radius, s))) return rc;
    // the computed parity goes to scratch a piece at a time: a 3 GiB shard set needs 1 GiB of it, not 12 GiB
    const size_t piece = std::min(n, size_t(256) << 20);
    struct Scratch {  // stream-ordered: freed after the work queued on s, on every exit path
        uint8_t* p = nullptr;
        cudaStream_t s;
        ~Scratch() {
            if (p) cudaFreeAsync(p, s);
        }
    } scratch{nullptr, s};
    if (piece) SWEC_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&scratch.p), size_t(m) * piece, s));
    for (size_t off = 0; off < n; off += piece) {
        const size_t len = std::min(piece, n - off);
        const uint8_t* in[SWEC_MAX_SHARDS];
        const uint8_t* stored[SWEC_MAX_SHARDS];
        uint8_t* comp[SWEC_MAX_SHARDS];
        for (int i = 0; i < k; i++) in[i] = sh[i] + off;
        for (int p = 0; p < m; p++) {
            comp[p] = scratch.p + size_t(p) * piece;
            stored[p] = sh[k + p] + off;
        }
        if ((rc = e->apply(rows, in, comp, len, Layout{}, s))) return rc;
        if ((rc = locator.launch(comp, stored, len, int64_t(off), s))) return rc;
    }
    SWEC_CUDA(cudaStreamSynchronize(s));
    return locator.collect(report, ranges, ranges_cap, n_ranges);
}

int swec_stream_synchronize(swec_encoder* e, void* stream) {
    if (!e) return fail(SWEC_ERR_INVALID_ARG, "NULL encoder");
    int rc = e->ensure_device();
    if (rc) return rc;
    SWEC_CUDA(cudaStreamSynchronize(pick_stream(e, stream)));
    return SWEC_OK;
}

// ---- pinned memory, measurement helpers

void* swec_alloc_pinned(size_t bytes) { return swec_alloc_pinned_for_device(-1, bytes); }

void* swec_alloc_pinned_for_device(int device, size_t bytes) {
    void* p = pinned_alloc(device, bytes);
    if (!p) set_last_error("pinned host allocation failed");
    return p;
}

void swec_free_pinned(void* p) { pinned_free(p); }

int swec_synth_fill_device(int device, void* dst, uint64_t byte_offset, size_t bytes, uint64_t seed, void* stream) {
    if (!dst || (byte_offset & 7) || (bytes & 7) || (reinterpret_cast<uintptr_t>(dst) & 7))
        return fail(SWEC_ERR_INVALID_ARG, "synth fill needs 8-byte aligned offset, size and pointer");
    SWEC_CUDA(cudaSetDevice(device));
    SWEC_CUDA(launch_synth(dst, byte_offset, bytes, seed, static_cast<cudaStream_t>(stream)));
    return SWEC_OK;
}

int swec_digest_device(int device, const void* src, size_t bytes, uint64_t* digest, void* stream) {
    if (!src || !digest) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    SWEC_CUDA(cudaSetDevice(device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    u64* d = nullptr;
    SWEC_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&d), 8, s));
    cudaError_t e = launch_digest(src, bytes, d, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(digest, d, 8, cudaMemcpyDeviceToHost, s);
    cudaFreeAsync(d, s);
    if (e != cudaSuccess) return cuda_fail(e, "digest");
    SWEC_CUDA(cudaStreamSynchronize(s));
    return SWEC_OK;
}

}  // extern "C"
