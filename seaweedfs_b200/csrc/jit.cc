// seaweedfs_b200/csrc/jit.cc — run-time specialisation of the Horner kernel for a given matrix.
//
// Reconstruct matrices depend on which shards survived (1001 ten-of-fourteen subsets for
// RS(10,4)), so they cannot all be compiled ahead of time.  The same generator that produced the
// AOT encode kernel (codegen.cc) emits the straight-line combine() for the fused decode matrix;
// NVRTC compiles it for sm_90a (≈0.3 s, once per matrix per process) and the cubin is loaded
// through the runtime's library API.  This is the GPU analogue of klauspost's cached inversion
// tree / the Rust twin's LRU of decode matrices (core.rs:25,700-734): the cache holds kernels.
//
// NVRTC is dlopen'ed so that libswec.so itself has no load-time dependency beyond cudart; if it
// cannot be found the engine uses the shared-memory table kernel instead (still on the GPU).
//
// The cache outlives the process: every compiled cubin is also written to an on-disk cache
// ($SWEC_CACHE_DIR, else $XDG_CACHE_HOME/swec, else ~/.cache/swec; SWEC_NO_DISK_CACHE=1 turns it off), named by a
// hash of the complete generated source, the target architecture and the CUDA runtime version.  A second process —
// or a volume server without libnvrtc — loads a previously seen erasure pattern in a few milliseconds instead of
// compiling for ~0.3 s.  The 15 most common patterns never get here at all: they are compiled with the library
// (aot_recon.cu).
#include <dlfcn.h>
#include <fcntl.h>
#include <nvrtc.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <map>
#include <mutex>
#include <thread>

#include "codegen.h"
#include "engine.h"

namespace swec {

static const char kDeviceCommonSrc[] =
#include "device_common_src.inc"
    ;

struct JitKernel {
    int threads = 256, unroll = 1;  // launch shape the kernel was specialised for
    cudaLibrary_t lib = nullptr;
    cudaKernel_t flat = nullptr, blocked = nullptr;
    CodegenStats stats;
};

namespace {

struct Nvrtc {
    void* handle = nullptr;
    decltype(&nvrtcCreateProgram) create = nullptr;
    decltype(&nvrtcCompileProgram) compile = nullptr;
    decltype(&nvrtcGetCUBINSize) cubin_size = nullptr;
    decltype(&nvrtcGetCUBIN) cubin = nullptr;
    decltype(&nvrtcGetProgramLogSize) log_size = nullptr;
    decltype(&nvrtcGetProgramLog) log = nullptr;
    decltype(&nvrtcDestroyProgram) destroy = nullptr;
    bool ok = false;
};

Nvrtc& nvrtc() {
    static Nvrtc n = [] {
        Nvrtc r;
        if (getenv("SWEC_NO_JIT")) return r;
        const char* names[] = {"libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so",
                               "/usr/local/cuda/lib64/libnvrtc.so"};
        for (const char* nm : names) {
            r.handle = dlopen(nm, RTLD_NOW | RTLD_LOCAL);
            if (r.handle) break;
        }
        if (!r.handle) return r;
#define SWEC_SYM(field, name) r.field = reinterpret_cast<decltype(r.field)>(dlsym(r.handle, name))
        SWEC_SYM(create, "nvrtcCreateProgram");
        SWEC_SYM(compile, "nvrtcCompileProgram");
        SWEC_SYM(cubin_size, "nvrtcGetCUBINSize");
        SWEC_SYM(cubin, "nvrtcGetCUBIN");
        SWEC_SYM(log_size, "nvrtcGetProgramLogSize");
        SWEC_SYM(log, "nvrtcGetProgramLog");
        SWEC_SYM(destroy, "nvrtcDestroyProgram");
#undef SWEC_SYM
        r.ok = r.create && r.compile && r.cubin_size && r.cubin && r.log_size && r.log && r.destroy;
        return r;
    }();
    return n;
}

struct JitEntry {
    enum State { kCold, kQueued, kCompiling, kReady, kFailed } state = kCold;
    int uses = 0;  // short-stream requests seen while cold
    std::shared_ptr<JitKernel> kernel;
};
struct JitRequest {
    Matrix rows;
    std::vector<uint8_t> key;
    int threads, unroll, device, variant;
    bool share_powers;
};
// Process-wide state.  Deliberately leaked (never destroyed): the compiler thread may still be
// finishing when static destructors run at process exit and must find the map and mutex alive.
struct JitGlobal {
    std::mutex mu;
    std::condition_variable cv;
    std::map<std::vector<uint8_t>, JitEntry> cache;
    std::deque<JitRequest> queue;  // background compiles, served by ONE worker thread
    std::thread worker;
    bool worker_started = false, stop = false;
};
JitGlobal& G() {
    static JitGlobal* g = new JitGlobal;
    return *g;
}
constexpr int kHotUses = 1;        // a matrix is worth a background compile from its first short use
constexpr size_t kMaxQueued = 16;  // beyond that the table kernel keeps serving

std::shared_ptr<JitKernel> build_kernel(const Matrix& rows, int threads, int unroll, int variant, bool share_powers);

void jit_worker_loop() {
    JitGlobal& g = G();
    std::unique_lock<std::mutex> lock(g.mu);
    for (;;) {
        g.cv.wait(lock, [&] { return g.stop || !g.queue.empty(); });
        if (g.stop) return;
        JitRequest rq = std::move(g.queue.front());
        g.queue.pop_front();
        g.cache[rq.key].state = JitEntry::kCompiling;
        lock.unlock();
        cudaSetDevice(rq.device);
        auto k = build_kernel(rq.rows, rq.threads, rq.unroll, rq.variant, rq.share_powers);
        lock.lock();
        g.cache[rq.key].kernel = k;
        g.cache[rq.key].state = k ? JitEntry::kReady : JitEntry::kFailed;
        g.cv.notify_all();
    }
}

// at exit: let the compile in progress (≤ ~1 s) land, then stop the worker before NVRTC/cudart go away
void jit_stop_at_exit() {
    JitGlobal& g = G();
    {
        std::lock_guard<std::mutex> lock(g.mu);
        g.stop = true;
        g.queue.clear();
    }
    g.cv.notify_all();
    if (g.worker.joinable()) g.worker.join();
}

}  // namespace

void jit_shutdown() { jit_stop_at_exit(); }

// everything the generated source depends on besides the matrix: a kernel cached under one key is the kernel of those options
static std::vector<uint8_t> jit_key(const Matrix& rows, int threads, int unroll, int variant, bool share_powers) {
    std::vector<uint8_t> key{uint8_t(rows.rows), uint8_t(rows.cols), uint8_t(threads / 64), uint8_t(unroll), uint8_t(variant),
                             uint8_t(share_powers)};
    key.insert(key.end(), rows.v.begin(), rows.v.end());
    return key;
}

bool jit_cached(swec_encoder_impl* enc, const Matrix& rows) {
    return enc->jit.count(jit_key(rows, int(g_opt_enc_threads.load()), int(g_opt_enc_unroll.load()), effective_xt_variant(),
                                  g_opt_jit_share_powers.load() != 0)) != 0;
}

// ---- on-disk cubin cache -------------------------------------------------------------------------------------
namespace {

bool cache_dir_trusted(const std::string& dir);

std::string disk_cache_dir() {
    if (getenv("SWEC_NO_DISK_CACHE")) return "";
    std::string dir;
    if (const char* d = getenv("SWEC_CACHE_DIR")) dir = d;
    else if (const char* x = getenv("XDG_CACHE_HOME"); x && *x) dir = std::string(x) + "/swec";
    else if (const char* h = getenv("HOME"); h && *h) dir = std::string(h) + "/.cache/swec";
    return !dir.empty() && cache_dir_trusted(dir) ? dir : "";
}

void mkdir_p(const std::string& dir) {
    for (size_t i = 1; i <= dir.size(); i++)
        if (i == dir.size() || dir[i] == '/') mkdir(dir.substr(0, i).c_str(), i == dir.size() ? 0700 : 0755);
}

// A cubin is executable code: only a directory that belongs to this user and that nobody else can write to is
// trusted as a cache (the same rule ssh applies to ~/.ssh).  Anything else disables the cache, never the engine.
bool cache_dir_trusted(const std::string& dir) {
    struct stat st;
    if (stat(dir.c_str(), &st) != 0) return true;  // does not exist yet: we create it 0700
    return S_ISDIR(st.st_mode) && st.st_uid == geteuid() && (st.st_mode & (S_IWGRP | S_IWOTH)) == 0;
}

// 128 bits of FNV-1a (two different offsets) over the text that determines the cubin
std::string cache_name(const std::string& src) {
    int rt = 0;
    cudaRuntimeGetVersion(&rt);
    const std::string all = "swec-cubin-v1|sm_90a|rt" + std::to_string(rt) + "|" + src;
    unsigned long long h1 = 0xcbf29ce484222325ull, h2 = 0x84222325cbf29ce4ull;
    for (unsigned char c : all) {
        h1 = (h1 ^ c) * 0x100000001b3ull;
        h2 = (h2 ^ (c + 0x9e)) * 0x100000001b3ull;
    }
    char buf[64];
    snprintf(buf, sizeof buf, "%016llx%016llx.cubin", h1, h2);
    return buf;
}

bool read_file(const std::string& path, std::vector<char>* out) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    fseek(f, 0, SEEK_END);
    const long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    out->resize(n > 0 ? size_t(n) : 0);
    const bool ok = n > 0 && fread(out->data(), 1, size_t(n), f) == size_t(n);
    fclose(f);
    return ok;
}

void write_file_atomic(const std::string& dir, const std::string& name, const std::vector<char>& data) {
    mkdir_p(dir);
    const std::string tmp = dir + "/." + name + "." + std::to_string(long(getpid())) + ".tmp";
    FILE* f = fopen(tmp.c_str(), "wb");
    if (!f) return;  // the cache is best effort
    const bool ok = fwrite(data.data(), 1, data.size(), f) == data.size();
    if (fclose(f) != 0 || !ok || rename(tmp.c_str(), (dir + "/" + name).c_str()) != 0) unlink(tmp.c_str());
}

std::atomic<unsigned long long> g_jit_compiles{0}, g_jit_disk_hits{0};

}  // namespace

unsigned long long jit_compile_count() { return g_jit_compiles.load(); }
unsigned long long jit_disk_hit_count() { return g_jit_disk_hits.load(); }

bool jit_available() { return nvrtc().ok || !disk_cache_dir().empty(); }

// the complete source of the two specialised kernels for `rows` (also the identity of the cached cubin)
static std::string jit_source(const Matrix& rows, int threads, int unroll, int variant, bool share_powers, CodegenStats* stats) {
    const std::string T = std::to_string(threads), U = std::to_string(unroll);
    std::string src = "#define SWEC_XT_VARIANT " + std::to_string(variant) + "\n";
    src += kDeviceCommonSrc;
    CodegenOptions copt;
    copt.share_powers = share_powers;  // off by default (kernels.h); the source text keys the cubin cache
    src += generate_combine(rows, "SwecJit", copt, stats);
    src +=
        "extern \"C\" __global__ void __launch_bounds__(" + T + ") swec_jit_flat(const __grid_constant__ SwecApplyParams p) {\n"
        "    swec_horner_body<SwecJit, false, " + U + ">(p);\n}\n"
        "extern \"C\" __global__ void __launch_bounds__(" + T + ") swec_jit_blocked(const __grid_constant__ SwecApplyParams p) {\n"
        "    swec_horner_body<SwecJit, true, " + U + ">(p);\n}\n";
    return src;
}

// cubin for `rows`: from the disk cache when this exact source was compiled before (by any process), else NVRTC
// (and into the cache).  No CUDA context needed.  *from_disk tells which.
static int compile_cubin(const Matrix& rows, int threads, int unroll, int variant, bool share_powers, std::vector<char>* cubin,
                         CodegenStats* stats,
                         bool* from_disk = nullptr, std::string* disk_path = nullptr) {
    if (rows.rows > SWEC_MAX_OUTPUTS) return fail(SWEC_ERR_JIT, "too many output rows for one specialised kernel");
    const std::string src = jit_source(rows, threads, unroll, variant, share_powers, stats);
    const std::string dir = disk_cache_dir(), name = dir.empty() ? "" : cache_name(src);
    if (from_disk) *from_disk = false;
    if (!dir.empty() && read_file(dir + "/" + name, cubin)) {
        if (from_disk) *from_disk = true;
        if (disk_path) *disk_path = dir + "/" + name;
        g_jit_disk_hits++;
        return SWEC_OK;
    }
    Nvrtc& n = nvrtc();
    if (!n.ok) return fail(SWEC_ERR_JIT, "NVRTC not available and this matrix is not in the cubin cache");
    // one NVRTC compile at a time (the background worker and an inline caller may otherwise overlap)
    static std::mutex& compile_mu = *new std::mutex;
    std::lock_guard<std::mutex> compile_lock(compile_mu);
    nvrtcProgram prog = nullptr;
    if (n.create(&prog, src.c_str(), "swec_jit.cu", 0, nullptr, nullptr) != NVRTC_SUCCESS)
        return fail(SWEC_ERR_JIT, "nvrtcCreateProgram failed");
    const char* opts[] = {"--gpu-architecture=sm_90a", "-std=c++17", "-lineinfo"};
    if (n.compile(prog, 3, opts) != NVRTC_SUCCESS) {
        size_t ls = 0;
        n.log_size(prog, &ls);
        std::string log(ls, '\0');
        if (ls) n.log(prog, &log[0]);
        n.destroy(&prog);
        return fail(SWEC_ERR_JIT, "NVRTC compile failed: " + log);
    }
    size_t cs = 0;
    n.cubin_size(prog, &cs);
    cubin->resize(cs);
    n.cubin(prog, cubin->data());
    n.destroy(&prog);
    g_jit_compiles++;
    if (!dir.empty()) write_file_atomic(dir, name, *cubin);
    return SWEC_OK;
}

namespace {
std::shared_ptr<JitKernel> build_kernel(const Matrix& rows, int threads, int unroll, int variant, bool share_powers) {
    for (int attempt = 0; attempt < 2; attempt++) {
        auto kernel = std::make_shared<JitKernel>();
        kernel->threads = threads;
        kernel->unroll = unroll;
        std::vector<char> cubin;
        bool from_disk = false;
        std::string disk_path;
        if (compile_cubin(rows, threads, unroll, variant, share_powers, &cubin, &kernel->stats, &from_disk, &disk_path) != SWEC_OK)
            return nullptr;
        cudaError_t e = cudaLibraryLoadData(&kernel->lib, cubin.data(), nullptr, nullptr, 0, nullptr, nullptr, 0);
        if (e == cudaSuccess) e = cudaLibraryGetKernel(&kernel->flat, kernel->lib, "swec_jit_flat");
        if (e == cudaSuccess) e = cudaLibraryGetKernel(&kernel->blocked, kernel->lib, "swec_jit_blocked");
        if (e == cudaSuccess) return kernel;
        cudaGetLastError();
        if (from_disk && attempt == 0) {  // a truncated / foreign file in the cache: drop it and compile
            unlink(disk_path.c_str());
            continue;
        }
        cuda_fail(e, "loading the specialised kernel");
        return nullptr;
    }
    return nullptr;
}

}  // namespace

// Long streams (wait = true) compile inline on the calling thread — ≈0.3 s, amortised.  Short ones never
// block: they are served by the table kernel, and a matrix that keeps coming back (degraded reads
// behind one dead server) is compiled once by the background worker and picked up when ready.
int jit_get(swec_encoder_impl* enc, const Matrix& rows, std::shared_ptr<JitKernel>* out, bool wait, bool hot) {
    const int threads = int(g_opt_enc_threads.load()), unroll = int(g_opt_enc_unroll.load());
    const int variant = effective_xt_variant();  // boost-clock or low-power step, by the device's recent load
    const bool share_powers = g_opt_jit_share_powers.load() != 0;  // read once: the key and a queued compile must agree
    const std::vector<uint8_t> key = jit_key(rows, threads, unroll, variant, share_powers);
    *out = nullptr;
    auto local = enc->jit.find(key);
    if (local != enc->jit.end()) {
        *out = local->second;
        return SWEC_OK;
    }
    if (!jit_available()) return fail(SWEC_ERR_JIT, "NVRTC not available and the cubin cache is off");
    JitGlobal& g = G();
    std::unique_lock<std::mutex> lock(g.mu);
    for (;;) {
        JitEntry& e = g.cache[key];
        if (e.state == JitEntry::kReady || e.state == JitEntry::kFailed) {
            enc->jit[key] = e.kernel;  // remember either outcome
            *out = e.kernel;
            return e.kernel ? SWEC_OK : SWEC_ERR_JIT;
        }
        if (!wait) {
            if (e.state == JitEntry::kCold && (++e.uses >= kHotUses || hot) && g.queue.size() < kMaxQueued && !g.stop) {
                int dev = 0;
                cudaGetDevice(&dev);
                e.state = JitEntry::kQueued;
                g.queue.push_back({rows, key, threads, unroll, dev, variant, share_powers});
                if (!g.worker_started) {
                    g.worker_started = true;
                    g.worker = std::thread(jit_worker_loop);
                    std::atexit(jit_stop_at_exit);
                }
                g.cv.notify_all();
            }
            return SWEC_OK;  // not ready: *out stays null
        }
        if (e.state == JitEntry::kCompiling) {  // someone else is on it
            g.cv.wait(lock);
            continue;
        }
        if (e.state == JitEntry::kQueued) {  // take it over from the queue
            for (auto it = g.queue.begin(); it != g.queue.end(); ++it)
                if (it->key == key) {
                    g.queue.erase(it);
                    break;
                }
        }
        e.state = JitEntry::kCompiling;
        lock.unlock();
        auto k = build_kernel(rows, threads, unroll, variant, share_powers);
        lock.lock();
        JitEntry& e2 = g.cache[key];
        e2.kernel = k;
        e2.state = k ? JitEntry::kReady : JitEntry::kFailed;
        g.cv.notify_all();
        enc->jit[key] = k;
        *out = k;
        return k ? SWEC_OK : SWEC_ERR_JIT;
    }
}

int jit_debug_compile(const Matrix& rows, size_t* cubin_bytes, int* xtime_steps, int* xor_ops) {
    std::vector<char> cubin;
    CodegenStats st;
    const int rc = compile_cubin(rows, int(g_opt_enc_threads.load()), int(g_opt_enc_unroll.load()), effective_xt_variant(),
                                 g_opt_jit_share_powers.load() != 0, &cubin, &st);
    if (cubin_bytes) *cubin_bytes = cubin.size();
    if (xtime_steps) *xtime_steps = st.xtime_steps;
    if (xor_ops) *xor_ops = st.xor_ops;
    return rc;
}

cudaError_t jit_launch(const JitKernel& k, const SwecApplyParams& p, bool blocked, cudaStream_t s) {
    if (p.nvec == 0) return cudaSuccess;
    int sms = 132, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const u64 per_cta = u64(k.threads) * u64(k.unroll);
    const u64 need = (p.nvec + per_cta - 1) / per_cta;
    const u64 cap = u64(sms) * u64(encode_ctas_per_sm());
    const unsigned grid = unsigned(need < cap ? need : cap);
    void* args[] = {const_cast<SwecApplyParams*>(&p)};
    note_kernel_work(double(p.nvec) * 16.0 * 14.0 / 3.0e12 * 1e3);  // ≈ k + r streams; feeds the power policy
    g_kernel_launches++;
    return cudaLaunchKernel(reinterpret_cast<const void*>(blocked ? k.blocked : k.flat), dim3(grid),
                            dim3(unsigned(k.threads)), args, 0, s);
}

}  // namespace swec
