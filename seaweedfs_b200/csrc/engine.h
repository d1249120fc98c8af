// seaweedfs_b200/csrc/engine.h — the encoder object behind the C ABI (include/swec.h).
//
// Mirrors what SeaweedFS holds as a reedsolomon.Encoder (ec_context.go:34-36): an immutable
// generator matrix plus, here, the device-side state needed to apply matrices on an H100:
// a stream, cached multiply tables / specialised kernels per matrix, and a small ring of pinned
// + device staging buffers for calls that arrive with host memory.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/swec.h"
#include "gf256.h"
#include "kernels.h"
#include "staging.h"

namespace swec {

void set_last_error(const std::string& msg);
const char* last_error();
int fail(int status, const std::string& msg);
int cuda_fail(cudaError_t e, const char* what);

#define SWEC_CUDA(call)                                     \
    do {                                                    \
        cudaError_t e__ = (call);                           \
        if (e__ != cudaSuccess) return cuda_fail(e__, #call); \
    } while (0)

size_t env_size(const char* name, size_t dflt);  // a positive integer from the environment, else dflt
size_t stage_slots();  // "stage_slots" (SWEC_STAGE_SLOTS): slots of every staging ring, at least 2
extern std::atomic<long> g_opt_stage_chunk;  // "stage_chunk" (SWEC_STAGE_CHUNK): largest piece per stream of a host call

// Device scratch in stream order: cudaMallocAsync on `s`, and freed after the work queued on s, on every exit path.
struct StreamScratch {
    void* p = nullptr;
    cudaStream_t s;
    explicit StreamScratch(cudaStream_t stream) : s(stream) {}
    StreamScratch(const StreamScratch&) = delete;
    ~StreamScratch() { if (p) cudaFreeAsync(p, s); }
    cudaError_t alloc(size_t bytes) { return cudaMallocAsync(&p, bytes, s); }
    template <class T> T* as() const { return static_cast<T*>(p); }
};

// Device memory that outlives any one stream: plain cudaMalloc, and cudaFree (on the current device) when the owner
// goes.  A failed alloc or upload leaves nothing to free by hand.
class DeviceBuffer {
  public:
    DeviceBuffer() = default;
    DeviceBuffer(DeviceBuffer&& o) noexcept : p_(o.p_), bytes_(o.bytes_) { o.p_ = nullptr; }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
        std::swap(p_, o.p_);
        std::swap(bytes_, o.bytes_);
        return *this;
    }
    ~DeviceBuffer() { if (p_) cudaFree(p_); }

    cudaError_t alloc(size_t bytes) {
        *this = DeviceBuffer();
        void* p = nullptr;
        const cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) p_ = p, bytes_ = bytes;
        return e;
    }
    // alloc, then copy host[0..n) on `s` and synchronise `s` (so work queued on s before is done too)
    template <class T> cudaError_t upload(const T* host, size_t n, cudaStream_t s) {
        cudaError_t e = alloc(n * sizeof(T));
        if (e == cudaSuccess) e = cudaMemcpyAsync(p_, host, n * sizeof(T), cudaMemcpyHostToDevice, s);
        return e == cudaSuccess ? cudaStreamSynchronize(s) : e;
    }
    // the whole buffer into *out, synchronously (cudaMemcpy)
    template <class T> cudaError_t read(std::vector<T>* out) const {
        out->resize(bytes_ / sizeof(T));
        return cudaMemcpy(out->data(), p_, out->size() * sizeof(T), cudaMemcpyDeviceToHost);
    }
    template <class T> T* as() const { return static_cast<T*>(p_); }

  private:
    void* p_ = nullptr;
    size_t bytes_ = 0;
};

// "file_direct_io" (SWEC_FILE_DIRECT): bit 0 = O_DIRECT reads of the .dat / shard inputs straight into the pinned
// ring, bit 1 = O_DIRECT writes of the shard outputs — the page cache is bypassed both ways (disk-backed volumes only;
// files that refuse O_DIRECT, tmpfs for one, and unaligned pieces silently take the buffered descriptor)
extern std::atomic<long> g_opt_file_direct_io;
void file_pipeline_trim();  // ec_files.cc: release staging rings parked between file-level calls

// device-resident multiply tables of one R×K matrix (R ≤ 4)
struct DeviceTables {
    DeviceBuffer compact;     // u32 [K][2][16]
    DeviceBuffer replicated;  // u32 [K][2][16][32]
};

struct JitKernel;  // jit.cc

struct Layout {  // how stream i / column x maps to memory; see SwecApplyParams
    bool blocked = false;
    uint64_t block_bytes = 0;
};

struct swec_encoder_impl {
    int k = 0, m = 0, device = -1;
    Matrix gen;
    bool rs10x4 = false;

    std::mutex mu;  // guards everything below
    cudaStream_t stream = nullptr;
    std::map<std::vector<uint8_t>, DeviceTables> tables;  // key: R, K, coefficients
    std::map<std::vector<uint8_t>, std::shared_ptr<JitKernel>> jit;  // same key
    StagingRing ring;  // (k+2m) streams of slot_chunk() bytes per slot
    // file pipelines never stall on a kernel compile: a cold matrix is served by the table kernel (100x faster
    // than the I/O around it) while the specialised kernel is built in the background and picked up when ready
    bool never_wait_for_jit = false;

    ~swec_encoder_impl();
    int ensure_device();  // cudaSetDevice + lazily create stream
    int ensure_slots(size_t chunk);
    size_t slot_chunk() const { return ring.bytes_per_slot / (size_t(k) + 2 * size_t(m)); }

    // out[r][x] = XOR_i rows[r][i] ⊗ in[i][x] on device memory, asynchronous on s.
    int apply(const Matrix& rows, const uint8_t* const* in, uint8_t* const* out, size_t n,
              const Layout& layout, cudaStream_t s);
    int get_tables(const Matrix& rows4, const DeviceTables** out, cudaStream_t s);
};

Matrix parity_rows(const swec_encoder_impl* e);  // the m parity rows of the generator

// true when run-time specialised kernels can be had: NVRTC loaded (SWEC_NO_JIT unset), or the on-disk cubin cache is on
bool jit_available();
unsigned long long jit_compile_count();   // NVRTC compiles done by this process
unsigned long long jit_disk_hit_count();  // kernels loaded from the on-disk cubin cache instead
// Specialised Horner kernel for `rows` on the current device (compiled once per matrix/process).
int jit_get(swec_encoder_impl* enc, const Matrix& rows, std::shared_ptr<JitKernel>* out, bool wait = true, bool hot = false);
int jit_debug_compile(const Matrix& rows, size_t* cubin_bytes, int* xtime_steps, int* xor_ops);
void jit_shutdown();  // stop the background compiler (idempotent); inline compiles keep working
bool jit_cached(swec_encoder_impl* enc, const Matrix& rows);
cudaError_t jit_launch(const JitKernel& k, const SwecApplyParams& p, bool blocked, cudaStream_t s);

}  // namespace swec

struct swec_encoder : swec::swec_encoder_impl {};
