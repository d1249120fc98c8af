// seaweedfs_b200/csrc/engine.cc — encoder object, matrix→kernel dispatch, reconstruct plans and the C ABI.
#include "engine.h"
#include "damage.h"
#include "host_seam.h"
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
std::atomic<long> g_opt_file_direct_io{long(env_size("SWEC_FILE_DIRECT", 0)) & 3};
std::atomic<long> g_opt_jit_enabled{1};
std::atomic<long> g_opt_jit_min_bytes{long(env_size("SWEC_JIT_MIN_BYTES", size_t(64) << 20))};

// ------------------------------------------------------------------ encoder lifetime

swec_encoder_impl::~swec_encoder_impl() {
    if (device < 0) return;
    if (cudaSetDevice(device) != cudaSuccess) return;  // the tables are freed after this body, on `device`
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

int swec_encoder_impl::get_tables(const Matrix& rows, const DeviceTables** out, cudaStream_t s) {
    const auto key = matrix_key(rows);
    auto it = tables.find(key);
    if (it != tables.end()) {
        *out = &it->second;
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
    SWEC_CUDA(t.compact.upload(compact.data(), compact.size(), s));
    SWEC_CUDA(t.replicated.upload(repl.data(), repl.size(), s));
    *out = &(tables[key] = std::move(t));
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
    // the table kernels, one launch per group of at most 4 rows: over the vectors, or over the byte tail
    auto table_groups = [&](bool byte_tail) -> int {
        for (int r0 = 0; r0 < R; r0 += 4) {
            const int rn = std::min(4, R - r0);
            Matrix sub(rn, K);
            memcpy(sub.v.data(), rows.row(r0), size_t(rn) * size_t(K));
            const DeviceTables* t;
            if (const int rc = get_tables(sub, &t, s)) return rc;
            SwecApplyParams p;
            fill(p, r0, rn, byte_tail ? tail_off : 0);
            if (byte_tail) SWEC_CUDA(launch_bytes_apply(p, t->compact.as<u32>(), K, rn, tail, s));
            else SWEC_CUDA(launch_table_apply(p, t->replicated.as<u32>(), K, rn, s));
        }
        return SWEC_OK;
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
                if (const int rc = table_groups(false)) return rc;
            }
        }
    }
    return tail ? table_groups(true) : SWEC_OK;
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
        case SWEC_ERR_UNCORRECTABLE: return "damage that cannot be corrected remains";
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

int swec_encode_device(swec_encoder* e, const void* const* data, void* const* parity, size_t n, void* stream) {
    if (!e || !data || !parity) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    std::lock_guard<std::mutex> lock(e->mu);
    int rc = e->ensure_device();
    if (rc) return rc;
    return e->apply(parity_rows(e), reinterpret_cast<const uint8_t* const*>(data),
                    reinterpret_cast<uint8_t* const*>(parity), n, Layout{}, static_cast<cudaStream_t>(stream));
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
    return e->apply(p.fused, ins, outs, n, Layout{}, static_cast<cudaStream_t>(stream));
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
                    Layout{}, static_cast<cudaStream_t>(stream));
}

int swec_encode_volume_device(swec_encoder* e, const void* dat_v, int64_t dat_size, int64_t large, int64_t small,
                              void* const* parity, void* stream) {
    if (!e || !dat_v || !parity || dat_size < 0 || large <= 0 || small <= 0)
        return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    const uint8_t* dat = static_cast<const uint8_t*>(dat_v);
    const int k = e->k, m = e->m;
    for (int p = 0; p < m; p++)
        if (!parity[p]) return fail(SWEC_ERR_INVALID_ARG, "NULL parity shard");
    std::lock_guard<std::mutex> lock(e->mu);
    int rc = e->ensure_device();
    if (rc) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
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
        // the blocked kernels read and write whole 16-byte vectors: every block and every parity stream must be aligned
        bool vec_ok = horner && block % 16 == 0 && (reinterpret_cast<uintptr_t>(base) & 15) == 0;
        for (int p = 0; p < m && vec_ok; p++) vec_ok = ((reinterpret_cast<uintptr_t>(parity[p]) + uint64_t(poff)) & 15) == 0;
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
        StreamScratch row(s);
        SWEC_CUDA(row.alloc(size_t(g.small_row())));
        SWEC_CUDA(cudaMemsetAsync(row.p, 0, size_t(g.small_row()), s));
        SWEC_CUDA(cudaMemcpyAsync(row.p, dat + g.tail_dat_offset(), size_t(g.tail), cudaMemcpyDeviceToDevice, s));
        rc = region(row.as<uint8_t>(), small, 1, g.tail_shard_offset());
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
    cudaStream_t s = static_cast<cudaStream_t>(stream);
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
    cudaStream_t s = static_cast<cudaStream_t>(stream);
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

}  // extern "C"

namespace {

// The device-level damage and checked calls: per piece, one apply of plan.fused from the information shards, the check
// rows into scratch and the rebuilt rows into the caller's buffers, then (c >= 1) the initialised locator; returns once
// the stream is done.  The computed check rows go to scratch a piece at a time: a 3 GiB shard set needs 1 GiB of it,
// not 12 GiB.  A data byte corrected in a piece has already been encoded, and no later piece reads it.  `fixer` (may be
// NULL): a correcting locator over plan.checks() that runs on each piece after `locator`, correcting the information and
// check shards in place.
int locate_pieces(swec_encoder* e, const CheckedPlan& plan, uint8_t* const* sh, size_t n, DamageLocator& locator,
                  cudaStream_t s, DamageLocator* fixer = nullptr) {
    const int k = e->k, c = plan.c();
    const size_t piece = std::min(n, size_t(256) << 20);
    StreamScratch scratch(s);
    if (piece && c > 0) SWEC_CUDA(scratch.alloc(size_t(c) * piece));
    for (size_t off = 0; off < n && !plan.outs.empty(); off += piece) {
        const size_t len = std::min(piece, n - off);
        const uint8_t* in[SWEC_MAX_SHARDS];
        uint8_t* at[SWEC_MAX_SHARDS];  // the shards at their locator positions: information, then check shards
        uint8_t* comp[SWEC_MAX_SHARDS];
        for (int j = 0; j < k; j++) in[j] = at[j] = sh[plan.info[size_t(j)]] + off;
        for (int i = 0; i < c; i++) {
            at[k + i] = sh[plan.check(i)] + off;
            comp[plan.check_rows[size_t(i)]] = scratch.as<uint8_t>() + size_t(i) * piece;
        }
        for (int o : plan.rebuilt_rows) comp[o] = sh[plan.outs[size_t(o)]] + off;
        int rc = e->apply(plan.fused, in, comp, len, Layout{}, s);
        if (rc == SWEC_OK && c > 0) rc = locator.launch(comp, at, len, int64_t(off), s);
        if (rc == SWEC_OK && fixer) {
            uint8_t* checks[SWEC_MAX_SHARDS];  // the computed check rows, in check order
            for (int i = 0; i < c; i++) checks[i] = comp[plan.check_rows[size_t(i)]];
            rc = fixer->launch(checks, at, len, int64_t(off), s);
        }
        if (rc) return rc;
    }
    SWEC_CUDA(cudaStreamSynchronize(s));
    return SWEC_OK;
}

// swec_locate_damage_device, and with `correct` swec_correct_damage_device: the shards are written only then.
int damage_device(swec_encoder* e, const void* const* shards, size_t n, int radius, bool correct, const DamageOut& out,
                  void* stream) {
    if (!e || !shards) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    int rc;
    if ((rc = out.check()) || (rc = check_radius(radius, 1, e->m))) return rc;
    for (int i = 0; i < e->k + e->m; i++)
        if (!shards[i]) return fail(SWEC_ERR_INVALID_ARG, "NULL shard");
    uint8_t* const* sh = reinterpret_cast<uint8_t* const*>(const_cast<void* const*>(shards));
    const CheckedPlan plan = CheckedPlan::all_present(e->gen, e->k);
    std::lock_guard<std::mutex> lock(e->mu);
    if ((rc = e->ensure_device())) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DamageLocator locator;
    if ((rc = locator.init(plan.fused, int64_t(n), radius, s, correct))) return rc;
    if ((rc = locate_pieces(e, plan, sh, n, locator, s))) return rc;
    return locator.collect(out);
}

}  // namespace

extern "C" {

int swec_locate_damage_device(swec_encoder* e, const void* const* shards, size_t n, int radius, swec_damage_report* report,
                              swec_damage_range* ranges, int ranges_cap, int* n_ranges, void* stream) {
    return damage_device(e, shards, n, radius, false, {report, ranges, ranges_cap, n_ranges}, stream);
}

int swec_correct_damage_device(swec_encoder* e, void* const* shards, size_t n, int radius, swec_damage_report* report,
                               swec_damage_range* ranges, int ranges_cap, int* n_ranges, void* stream) {
    return damage_device(e, shards, n, radius, true, {report, ranges, ranges_cap, n_ranges}, stream);
}

}  // extern "C"

namespace {

// swec_reconstruct_checked_device, and with `decode` swec_decode_data_checked_device.  The first k present shards are
// the information set; the other c present shards are re-encoded from it into scratch and checked, and the missing
// shards are rebuilt into the caller's buffers by the same apply, then cleared of the errors the locator finds in the
// information set.  The rebuild reads every present shard and rebuilds every missing one.  The decode rebuilds only the
// missing data shards and also corrects the present data shards in place; parity shards are only read, and a missing
// one needs no buffer.  The heal (swec_heal_device, `heal`) is the rebuild that also corrects every present shard in
// place: after the rebuilding locator, each piece goes through a correcting locator over P', which decodes the same
// syndromes at the same radius and so writes back exactly the errors the report blames.  Its own report is dropped.
int checked_device(swec_encoder* e, void* const* shards, const uint8_t* present, size_t n, int radius, bool decode,
                   const DamageOut& out, void* stream, bool heal = false) {
    if (!e || !shards || !present) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    int rc;
    if ((rc = out.check()) || (rc = check_radius(radius, 0))) return rc;
    const int k = e->k, total = e->k + e->m;
    CheckedPlan plan;
    if (!plan.build(e->gen, k, present, decode)) return fail(SWEC_ERR_TOO_FEW_SHARDS, "fewer than data_shards shards present");
    for (int i = 0; i < total; i++)
        if (!shards[i] && (present[i] || i < k || !decode))
            return fail(SWEC_ERR_INVALID_ARG, present[i] ? "NULL shard" : "missing shard has no buffer");
    std::lock_guard<std::mutex> lock(e->mu);
    if ((rc = e->ensure_device())) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DamageLocator locator;
    if (plan.c() > 0 && (rc = locator.init_rebuild(plan, int64_t(n), radius, s))) return rc;
    DamageLocator fixer;  // radius 0 decodes nothing, so it corrects nothing
    const bool fix = heal && plan.radius(radius) > 0;
    if (fix && (rc = fixer.init(plan.checks(), int64_t(n), plan.radius(radius), s, /*correct=*/true))) return rc;
    if ((rc = locate_pieces(e, plan, reinterpret_cast<uint8_t* const*>(shards), n, locator, s, fix ? &fixer : nullptr)))
        return rc;
    if (plan.c() == 0) {  // every present shard is an information shard: nothing to check
        out.unchecked();
        return SWEC_OK;
    }
    return locator.collect(out);
}

}  // namespace

extern "C" {

int swec_reconstruct_checked_device(swec_encoder* e, void* const* shards, const uint8_t* present, size_t n, int radius,
                                    swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges,
                                    void* stream) {
    return checked_device(e, shards, present, n, radius, false, {report, ranges, ranges_cap, n_ranges}, stream);
}

int swec_decode_data_checked_device(swec_encoder* e, void* const* shards, const uint8_t* present, size_t n, int radius,
                                    swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges,
                                    void* stream) {
    return checked_device(e, shards, present, n, radius, true, {report, ranges, ranges_cap, n_ranges}, stream);
}

int swec_heal_device(swec_encoder* e, void* const* shards, const uint8_t* present, size_t n, int radius,
                     swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges, void* stream) {
    return checked_device(e, shards, present, n, radius, false, {report, ranges, ranges_cap, n_ranges}, stream, true);
}

int swec_stream_synchronize(swec_encoder* e, void* stream) {
    if (!e) return fail(SWEC_ERR_INVALID_ARG, "NULL encoder");
    int rc = e->ensure_device();
    if (rc) return rc;
    SWEC_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
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
    StreamScratch d(s);
    SWEC_CUDA(d.alloc(8));
    SWEC_CUDA(launch_digest(src, bytes, d.as<u64>(), s));
    SWEC_CUDA(cudaMemcpyAsync(digest, d.p, 8, cudaMemcpyDeviceToHost, s));
    SWEC_CUDA(cudaStreamSynchronize(s));
    return SWEC_OK;
}

}  // extern "C"
