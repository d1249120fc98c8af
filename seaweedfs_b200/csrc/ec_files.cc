// seaweedfs_b200/csrc/ec_files.cc — file-level entry points: the GPU twins of
//   generateEcFiles / encodeDatFile / encodeData / encodeDataOneBatch
//       (weed/storage/erasure_coding/ec_encoder.go:110-128, 202-222, 248-278, 280-321)
//   generateMissingEcFiles / rebuildEcFiles / findShardFile      (ec_encoder.go:131-200, 323-377)
//   WriteDatFile                                                (ec_decoder.go:176-223)
// Same files, same bytes, same error points; different schedule.  The reference runs
// read → Encode → write serially in 256 KiB batches on one goroutine.  Here a reader stages multi-MiB
// stripes into pinned slots, the GPU turns each slot round on its own stream (H2D, kernel, D2H)
// and a writer thread drains finished slots with pwrite at explicit shard offsets, so disk reads,
// PCIe, the kernel and disk writes all overlap.  Batch size is result-neutral (the code is
// column-wise), so buffer_size is only validated the way the reference does.
#include <errno.h>
#include <fcntl.h>
#include <linux/falloc.h>
#include <sys/stat.h>
#include <sys/vfs.h>
#include <unistd.h>

#include <algorithm>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <memory>
#include <thread>
#include <time.h>

#include "damage.h"
#include "engine.h"
#include "io_pool.h"
#include "needle_damage.h"
#include "volume_format.h"

namespace swec {
namespace {

int io_fail(const std::string& what) { return fail(SWEC_ERR_IO, what + ": " + strerror(errno)); }

// The first failure of work spread over several threads.  Error texts are thread-local, so the status keeps the
// last_error() text of the thread that reported it, and get() hands both to the thread that owns the work.
class FirstError {
  public:
    int report(int rc) {  // any thread; returns rc
        std::lock_guard<std::mutex> lk(mu_);
        if (rc && !rc_) {
            rc_ = rc;
            text_ = last_error();
        }
        return rc;
    }
    int fail(int rc, const std::string& msg) { return report(swec::fail(rc, msg)); }
    int status() {
        std::lock_guard<std::mutex> lk(mu_);
        return rc_;
    }
    int get() {  // the first status, its text set as the calling thread's last error
        std::lock_guard<std::mutex> lk(mu_);
        if (rc_) set_last_error(text_);
        return rc_;
    }

  private:
    std::mutex mu_;
    int rc_ = 0;
    std::string text_;
};

// Reserving extents pays on disk filesystems (once instead of 14 files growing 8 MiB at a time) and costs on tmpfs,
// where it zero-fills every page that the writers overwrite a moment later.  The reservation must NOT change the
// visible file size: DiskLocation.validateEcVolume (disk_location_ec.go:455-530) and rebuildEcFiles' equal-length
// check recognise an interrupted encode by its short shards, so a killed run has to leave short files, not
// full-size files of zeros — hence FALLOC_FL_KEEP_SIZE (reserve_extents), never posix_fallocate.
bool worth_preallocating(int fd) {
    if (getenv("SWEC_NO_FALLOCATE")) return false;
    struct statfs fs;
    if (fstatfs(fd, &fs) != 0) return true;
    return fs.f_type != 0x01021994 /* TMPFS_MAGIC */ && fs.f_type != 0x858458f6 /* RAMFS_MAGIC */;
}

// a second descriptor on the same file with O_DIRECT, or -1 (tmpfs and friends refuse it; so may the caller's option)
int open_direct(const std::string& path, int flags, bool wanted) {
    if (!wanted) return -1;
    const int fd = open(path.c_str(), flags | O_DIRECT);
    if (fd < 0) errno = 0;
    return fd;
}
inline bool direct_ok(int dfd, int64_t off, size_t len, const void* buf) {
    return dfd >= 0 && ((uint64_t(off) | uint64_t(len) | reinterpret_cast<uintptr_t>(buf)) & 4095) == 0;
}

struct FdSet {
    std::vector<int> fds;
    int keep(int fd) {  // closed with the set unless negative; returns fd
        if (fd >= 0) fds.push_back(fd);
        return fd;
    }
    ~FdSet() {
        for (int fd : fds)
            if (fd >= 0) close(fd);
    }
};

// fill bytes [dst_off, dst_off+len) of the slot's stream `stream` from fd@off (zero past EOF)
// dfd: the same file opened O_DIRECT (-1 = none): used when offset, length and buffer are all 4 KiB aligned
struct ReadOp { int stream, fd; int64_t off; size_t dst_off, len; int dfd = -1; };
// drain bytes [src_off, src_off+len) of the slot's stream `stream` to fd@off
struct WriteOp { int stream, fd; int64_t off; size_t src_off, len; int dfd = -1; };
struct Item {
    size_t len = 0;
    int64_t shard_off = 0;  // shard offset of the item's first column
    std::vector<ReadOp> reads;
    std::vector<WriteOp> writes;
};

struct Slot {
    StagingSlot* buf;  // a slot of the pipeline's staging ring
    Item item;
};

// ONE I/O pool per process, shared by every file pipeline: concurrent volumes (the shell runs up to 10 at once) must not
// multiply the thread count — on an earlier GPU generation's hosts, 4 pipelines x 16 threads on a 16-core cgroup quota ran
// at less than half the rate of one volume alone (not re-measured on H100 hosts).  Size: the CPU time the process may actually use (cgroup quota,
// else the hardware concurrency), between 4 and 64; SWEC_IO_THREADS overrides.  Leaked on purpose, like the other
// process-wide helpers: threads must not be joined from static destructors.
size_t usable_cpus() {
    size_t n = std::max(1u, std::thread::hardware_concurrency());
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {  // cgroup v2: "<quota|max> <period>"
        char q[32] = {0};
        long long period = 0;
        if (fscanf(f, "%31s %lld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0)
            n = std::min<size_t>(n, size_t(std::max<long long>(1, (atoll(q) + period - 1) / period)));
        fclose(f);
    } else {
        long long quota = -1, period = 0;
        if (FILE* g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) {
            if (fscanf(g, "%lld", &quota) != 1) quota = -1;
            fclose(g);
        }
        if (FILE* g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) {
            if (fscanf(g, "%lld", &period) != 1) period = 0;
            fclose(g);
        }
        if (quota > 0 && period > 0) n = std::min<size_t>(n, size_t(std::max<long long>(1, (quota + period - 1) / period)));
    }
    return n;
}
IoPool& file_io_pool() {
    static IoPool* pool = new IoPool(env_size("SWEC_IO_THREADS", std::min<size_t>(64, std::max<size_t>(4, usable_cpus()))));
    return *pool;
}

// Slot pitch of a pipeline over streams of `span` bytes: the configured chunk (8 MiB), or less for a shorter span, in
// whole 256-byte units.  Parked rings are matched by slot size, so every file-level call takes its chunk from here.
size_t file_chunk(int64_t span) {
    const int64_t cap = int64_t(env_size("SWEC_FILE_CHUNK", size_t(8) << 20));
    return std::max<size_t>(256, (size_t(std::min<int64_t>(cap, std::max<int64_t>(span, 1))) + 255) & ~size_t(255));
}

// Staging rings outlive a call: pinning (mmap + mbind + cudaHostRegister) and un-pinning 3 x 14 x 8 MiB costs
// 0.1-2 s per call, as much as the pipeline itself spends on an 8 GiB volume.  A volume
// server encodes volume after volume, so finished pipelines park their ring here (per device, slot size and slot
// count, a few at most) and the next call picks it up.  swec_shutdown() releases them.
std::mutex& parked_mu() {
    static std::mutex* m = new std::mutex;
    return *m;
}
std::vector<StagingRing>& parked_rings() {
    static std::vector<StagingRing>* c = new std::vector<StagingRing>;  // leaked on purpose: no CUDA calls in static destructors
    return *c;
}
constexpr size_t kMaxParkedRings = 4;

// wall-clock breakdown of one pipeline run, printed to stderr as JSON when SWEC_PIPE_STATS is set
struct PipeStats {
    double setup = 0, prealloc = 0, wait_slot = 0, read = 0, enqueue = 0, wait_gpu = 0, write = 0, total = 0;
    int items = 0;
    static double now() {
        struct timespec t;
        clock_gettime(CLOCK_MONOTONIC, &t);
        return double(t.tv_sec) + double(t.tv_nsec) * 1e-9;
    }
};

// The outputs' final size is known up front: reserve it (best effort, one I/O thread per file), so that the writers
// fill extents that already exist instead of growing every file 8 MiB at a time under the filesystem's allocation lock.
// Returns the seconds spent reserving: 0 where it does not pay.
double reserve_extents(const std::vector<int>& outs, int64_t size) {
    if (size <= 0 || !worth_preallocating(outs[0])) return 0;
    const double t0 = PipeStats::now();
    file_io_pool().parallel_for(int(outs.size()), [&](int i) -> int {
        if (fallocate(outs[size_t(i)], FALLOC_FL_KEEP_SIZE, 0, off_t(size)) != 0) errno = 0;  // the length stays as written
        return 0;
    });
    return PipeStats::now() - t0;
}

// K input streams, then `stored` streams read from disk, then R computed streams per slot, pitch = chunk bytes.
class FilePipeline {
  public:
    // What runs on each item after the apply: the R computed rows, the slot's K + stored read streams, the item's
    // columns and shard offset, and the index of its slot, in the slot's stream order.
    using Step = std::function<int(uint8_t* const* computed, uint8_t* const* shards, size_t len, int64_t base, int slot,
                                   cudaStream_t s)>;
    PipeStats stats;
    // Without a step the R computed rows come back to be written.  With one, the streams the item writes (corrected,
    // rebuilt or computed) come back, once each, after the step.
    FilePipeline(swec_encoder* enc, const Matrix& rows, size_t chunk, int stored = 0, Step step = {})
        : enc_(enc), rows_(rows), chunk_(chunk), stored_(stored), step_(std::move(step)) {}
    ~FilePipeline() { shutdown(); }

    int start() {
        t_begin_ = PipeStats::now();
        enc_->never_wait_for_jit = !getenv("SWEC_FILE_JIT_WAIT");
        int rc = enc_->ensure_device();
        if (rc) return rc;
        const size_t nslots = stage_slots();
        const size_t streams = size_t(rows_.cols + stored_ + rows_.rows);
        // one size for every kind of pipeline of this code on this device (generate: k+m streams, rebuild: k + missing,
        // verify: k+2m, checked rebuild: k + c + m <= k+2m), so that a parked ring fits whichever call comes next
        const size_t slot_bytes = std::max(streams, size_t(enc_->k + 2 * enc_->m)) * chunk_;
        {
            std::lock_guard<std::mutex> lk(parked_mu());
            auto& parked = parked_rings();
            for (size_t i = 0; i < parked.size(); i++)
                if (parked[i].device == enc_->device && parked[i].bytes_per_slot == slot_bytes && parked[i].slots.size() == nslots) {
                    ring_ = std::move(parked[i]);
                    parked.erase(parked.begin() + long(i));
                    break;
                }
        }
        if (ring_.slots.empty() && (rc = ring_.allocate(enc_->device, nslots, slot_bytes))) return rc;
        for (StagingSlot& b : ring_.slots) slots_.push_back({&b, Item{}});
        for (Slot& s : slots_) free_.push_back(&s);
        io_ = &file_io_pool();
        writer_ = std::thread([this] { writer_loop(); });
        started_ = true;
        stats.setup = PipeStats::now() - t_begin_;  // printed only for a pipeline that started
        return SWEC_OK;
    }

    // blocking: read the item's inputs, queue the GPU work, hand the slot to the writer
    int submit(Item&& item) {
        Slot* s = nullptr;
        double t0 = PipeStats::now();
        {
            std::unique_lock<std::mutex> lk(mu_);
            cv_.wait(lk, [&] { return !free_.empty() || first_.status(); });
            if (const int rc = first_.status()) return rc;
            s = free_.front();
            free_.pop_front();
        }
        StagingSlot& b = *s->buf;
        double t1 = PipeStats::now();
        stats.wait_slot += t1 - t0;
        stats.items++;
        const int K = rows_.cols, R = rows_.rows;
        const size_t len = item.len;
        // Every pread is cut into pieces of at most io_piece_ bytes so that ONE stripe keeps the whole I/O pool busy
        // (k preads of 8 MiB are only k tasks; a thread copies 2-3 GB/s out of the page cache into cache-cold memory).
        struct Piece { int op; size_t off, len; };
        std::vector<Piece> rpieces;
        for (size_t i = 0; i < item.reads.size(); i++)
            for (size_t o = 0; o < item.reads[i].len; o += io_piece_)
                rpieces.push_back({int(i), o, std::min(io_piece_, item.reads[i].len - o)});
        const std::function<int(int)> read_one = [&](int idx) -> int {
            const Piece& pc = rpieces[size_t(idx)];
            const ReadOp& r = item.reads[size_t(pc.op)];
            uint8_t* dst = b.host + size_t(r.stream) * chunk_ + r.dst_off + pc.off;
            const int64_t off = r.off + int64_t(pc.off);
            const size_t len = pc.len;
            // O_DIRECT: the device DMAs straight into the pinned slot; short counts only happen at EOF, where the
            // remainder (unaligned now) continues on the buffered descriptor
            const int fd0 = direct_ok(r.dfd, off, len, dst) ? r.dfd : r.fd;
            size_t got = 0;
            while (got < len) {
                const int fd = (fd0 == r.dfd && direct_ok(r.dfd, off + int64_t(got), len - got, dst + got)) ? r.dfd : r.fd;
                const ssize_t n = pread(fd, dst + got, len - got, off_t(off + int64_t(got)));
                if (n < 0) {
                    if (errno == EINTR) continue;
                    return first_.report(io_fail("pread"));
                }
                if (n == 0) break;  // EOF: the rest reads as zero (ec_encoder.go:258-262)
                got += size_t(n);
            }
            if (got < len) memset(dst + got, 0, len - got);
            return SWEC_OK;
        };
        if (const int rrc = io_->parallel_for(int(rpieces.size()), read_one)) return set_error(rrc, s);
        t0 = PipeStats::now();
        stats.read += t0 - t1;
        if (cudaSetDevice(enc_->device) != cudaSuccess) return set_error(fail(SWEC_ERR_CUDA, "cudaSetDevice"), s);
        cudaError_t e = cudaSuccess;
        const uint8_t* din[SWEC_MAX_SHARDS];
        uint8_t* dout[SWEC_MAX_SHARDS];
        for (int i = 0; i < K; i++) din[i] = b.dev + size_t(i) * chunk_;
        const int nin = K + stored_;
        if (len == chunk_) {  // full slot: the input streams are contiguous — one DMA
            e = cudaMemcpyAsync(b.dev, b.host, size_t(nin) * chunk_, cudaMemcpyHostToDevice, b.stream);
        } else {
            for (int i = 0; i < nin && e == cudaSuccess; i++)
                e = cudaMemcpyAsync(b.dev + size_t(i) * chunk_, b.host + size_t(i) * chunk_, len, cudaMemcpyHostToDevice, b.stream);
        }
        if (e != cudaSuccess) return set_error(cuda_fail(e, "H2D"), s);
        for (int r = 0; r < R; r++) dout[r] = b.dev + size_t(K + stored_ + r) * chunk_;
        int rc;
        {
            std::lock_guard<std::mutex> lk(enc_->mu);
            rc = enc_->apply(rows_, din, dout, len, Layout{}, b.stream);
        }
        if (rc) return set_error(rc, s);
        if (step_) {
            uint8_t* shards[SWEC_MAX_SHARDS];
            for (int i = 0; i < K + stored_; i++) shards[i] = b.dev + size_t(i) * chunk_;
            if ((rc = step_(dout, shards, len, item.shard_off, int(s - slots_.data()), b.stream))) return set_error(rc, s);
            uint64_t back = 0;
            for (const WriteOp& w : item.writes) {
                if ((back >> w.stream) & 1) continue;
                back |= uint64_t(1) << w.stream;
                if (e == cudaSuccess)
                    e = cudaMemcpyAsync(b.host + size_t(w.stream) * chunk_, b.dev + size_t(w.stream) * chunk_, len,
                                        cudaMemcpyDeviceToHost, b.stream);
            }
        } else if (len == chunk_) {
            e = cudaMemcpyAsync(b.host + size_t(K) * chunk_, dout[0], size_t(R) * chunk_, cudaMemcpyDeviceToHost, b.stream);
        } else {
            for (int r = 0; r < R && e == cudaSuccess; r++)
                e = cudaMemcpyAsync(b.host + size_t(K + r) * chunk_, dout[r], len, cudaMemcpyDeviceToHost, b.stream);
        }
        if (e == cudaSuccess) e = cudaEventRecord(b.done, b.stream);
        if (e != cudaSuccess) return set_error(cuda_fail(e, "D2H"), s);
        s->item = std::move(item);
        {
            std::lock_guard<std::mutex> lk(mu_);
            inflight_.push_back(s);
        }
        cv_.notify_all();
        stats.enqueue += PipeStats::now() - t0;
        return SWEC_OK;
    }

    // wait for everything queued so far, or for the first error of submit(), the reads or the writes: returned, with
    // its text set as the calling thread's last error
    int finish() {
        {
            std::unique_lock<std::mutex> lk(mu_);
            cv_.wait(lk, [&] { return (inflight_.empty() && free_.size() == slots_.size()) || first_.status(); });
        }
        return first_.get();
    }

    void report(const char* what) {
        if (!getenv("SWEC_PIPE_STATS")) return;
        stats.total = PipeStats::now() - t_begin_;
        fprintf(stderr,
                "{\"pipe\": \"%s\", \"items\": %d, \"chunk\": %zu, \"total_s\": %.3f, \"setup_s\": %.3f, \"prealloc_s\": %.3f, "
                "\"reader\": {\"wait_slot_s\": %.3f, \"read_s\": %.3f, \"enqueue_s\": %.3f}, "
                "\"writer\": {\"wait_gpu_s\": %.3f, \"write_s\": %.3f}}\n",
                what, stats.items, chunk_, stats.total, stats.setup, stats.prealloc, stats.wait_slot, stats.read, stats.enqueue,
                stats.wait_gpu, stats.write);
    }

    void shutdown() {
        if (!started_) return;
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
        }
        cv_.notify_all();
        if (writer_.joinable()) writer_.join();
        io_ = nullptr;
        cudaSetDevice(enc_->device);
        bool healthy = first_.status() == 0;
        for (StagingSlot& b : ring_.slots)
            if (cudaStreamSynchronize(b.stream) != cudaSuccess) {
                cudaGetLastError();
                healthy = false;
            }
        free_.clear();
        inflight_.clear();
        slots_.clear();
        if (healthy && !ring_.slots.empty() && !getenv("SWEC_NO_RING_CACHE")) {  // park the ring for the next call
            std::lock_guard<std::mutex> lk(parked_mu());
            auto& parked = parked_rings();
            if (parked.size() < kMaxParkedRings) parked.push_back(std::move(ring_));  // leaves ring_ without slots
        }
        ring_.release();
        started_ = false;
    }

    size_t slot_count() const { return slots_.size(); }  // after start()

  private:
    // Every failure reaches first_ under mu_, here or in the writer loop, and a wake-up follows, so no waiter can test
    // first_ just before the report and then sleep through it.  I/O tasks report earlier, without mu_, to keep their
    // own text; the report under mu_ then finds the status taken.
    int set_error(int rc, Slot* s) {
        std::lock_guard<std::mutex> lk(mu_);
        first_.report(rc);
        if (s) free_.push_back(s);
        cv_.notify_all();
        return rc;
    }

    void writer_loop() {
        cudaSetDevice(enc_->device);
        for (;;) {
            Slot* s = nullptr;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return !inflight_.empty() || stop_; });
                if (inflight_.empty()) return;
                s = inflight_.front();
            }
            int rc = SWEC_OK;
            const double tw0 = PipeStats::now();
            if (cudaEventSynchronize(s->buf->done) != cudaSuccess) rc = fail(SWEC_ERR_CUDA, "cudaEventSynchronize failed in the shard writer");
            const double tw1 = PipeStats::now();
            stats.wait_gpu += tw1 - tw0;   // writer thread only
            if (!rc) {
                struct Piece { int op; size_t off, len; };
                std::vector<Piece> wpieces;
                // one task per shard file: buffered writes take the inode's lock exclusively, so pieces of the same
                // file would only queue behind each other (SWEC_FILE_WRITE_PIECE splits them anyway, for O_DIRECT devices)
                const size_t wpiece = std::max<size_t>(4096, env_size("SWEC_FILE_WRITE_PIECE", s->item.len ? s->item.len : 4096) & ~size_t(4095));
                for (size_t i = 0; i < s->item.writes.size(); i++)
                    for (size_t o = 0; o < s->item.writes[i].len; o += wpiece)
                        wpieces.push_back({int(i), o, std::min(wpiece, s->item.writes[i].len - o)});
                const std::function<int(int)> write_one = [&](int idx) -> int {
                    const Piece& pc = wpieces[size_t(idx)];
                    const WriteOp& w = s->item.writes[size_t(pc.op)];
                    const uint8_t* src = s->buf->host + size_t(w.stream) * chunk_ + w.src_off + pc.off;
                    const int64_t off = w.off + int64_t(pc.off);
                    size_t put = 0;
                    while (put < pc.len) {
                        const int fd = direct_ok(w.dfd, off + int64_t(put), pc.len - put, src + put) ? w.dfd : w.fd;
                        const ssize_t n = pwrite(fd, src + put, pc.len - put, off_t(off + int64_t(put)));
                        if (n < 0) {
                            if (errno == EINTR) continue;
                            return first_.report(io_fail("pwrite"));
                        }
                        put += size_t(n);
                    }
                    return SWEC_OK;
                };
                rc = io_->parallel_for(int(wpieces.size()), write_one);
                stats.write += PipeStats::now() - tw1;
            }
            {
                std::lock_guard<std::mutex> lk(mu_);
                inflight_.pop_front();
                free_.push_back(s);
                first_.report(rc);
            }
            cv_.notify_all();
        }
    }

    swec_encoder* enc_;
    Matrix rows_;
    size_t chunk_;
    const size_t io_piece_ = std::max<size_t>(4096, env_size("SWEC_FILE_IO_PIECE", size_t(2) << 20) & ~size_t(4095));
    double t_begin_ = 0;
    int stored_ = 0;  // streams read after the K inputs
    Step step_;
    StagingRing ring_;
    std::vector<Slot> slots_;  // one per ring slot
    std::deque<Slot*> free_, inflight_;
    std::mutex mu_;
    std::condition_variable cv_;
    std::thread writer_;
    IoPool* io_ = nullptr;  // the process-wide pool (not owned)
    FirstError first_;      // of submit(), the reader's and writer's I/O tasks and the writer
    bool stop_ = false, started_ = false;
};

// The step of the damage pipelines: the locator compares, and corrects or rebuilds, in the slot.
FilePipeline::Step locate_step(DamageLocator& locator) {
    return [&locator](uint8_t* const* computed, uint8_t* const* shards, size_t len, int64_t base, int, cudaStream_t s) {
        return locator.launch(computed, shards, len, base, s);
    };
}

}  // namespace

void file_pipeline_trim() {  // swec_shutdown(): release parked staging rings
    std::vector<StagingRing> rings;
    {
        std::lock_guard<std::mutex> lk(parked_mu());
        rings.swap(parked_rings());
    }
    for (StagingRing& r : rings) r.release();
}

}  // namespace swec

using namespace swec;

namespace {

struct EncoderFree {
    void operator()(swec_encoder* e) const { swec_encoder_free(e); }
};
using CallEncoder = std::unique_ptr<swec_encoder, EncoderFree>;

// the encoder of one file-level call, freed on every way out of it
int new_call_encoder(int k, int m, int device, CallEncoder* enc) {
    swec_encoder* e = nullptr;
    const int rc = swec_encoder_new(k, m, device, &e);
    enc->reset(e);
    return rc;
}

// findShardFile, opened read-only into `fds` (*fd = -1: no such shard) — with its O_DIRECT twin in *dfd when asked for
int open_shard(const std::string& b, const char* const* dirs, int ndirs, int i, FdSet* fds, int* fd, int* dfd = nullptr,
               bool direct = false) {
    *fd = -1;
    const std::string path = find_shard_file(b, dirs, ndirs, i);
    if (path.empty()) return SWEC_OK;
    if ((*fd = fds->keep(open(path.c_str(), O_RDONLY))) < 0) return io_fail("open " + path);
    if (dfd) *dfd = fds->keep(open_direct(path, O_RDONLY, direct));
    return SWEC_OK;
}

// Every shard of the set opened, all of one length: what a parity scrub needs (verify_ec_shards, ec_encoder.rs:177-278).
// The first problem in shard order wins.
int open_all_shards(const std::string& b, const char* const* dirs, int ndirs, int total, FdSet* fds, std::vector<int>* in,
                    int64_t* size) {
    in->assign(static_cast<size_t>(total), -1);
    *size = -1;
    for (int i = 0; i < total; i++) {
        int& fd = (*in)[size_t(i)];
        if (const int rc = open_shard(b, dirs, ndirs, i, fds, &fd)) return rc;
        if (fd < 0) return fail(SWEC_ERR_TOO_FEW_SHARDS, "verify needs all shards; missing " + shard_ext(i));
        if (const int rc = check_length(fd, size)) return rc;
    }
    return SWEC_OK;
}

// Every column of the shard set through a started verify pipeline; returns pipe.finish().
int scrub_columns(FilePipeline& pipe, const std::vector<int>& in, int64_t size, size_t chunk) {
    for (int64_t o = 0; o < size; o += int64_t(chunk)) {
        Item it;
        it.len = size_t(std::min<int64_t>(int64_t(chunk), size - o));
        it.shard_off = o;
        for (size_t i = 0; i < in.size(); i++) it.reads.push_back({int(i), in[i], o, 0, it.len});
        if (pipe.submit(std::move(it))) break;
    }
    return pipe.finish();
}

// Pass 2 of the damage calls, through a started pipeline: the union of pass 1's page `runs` as maximal spans, cut into
// items of at most `chunk` columns, each reading its columns from every shard (in_d: O_DIRECT twins, -1 = none).
// `add` adds what else an item needs (the repair: its writes) before it is submitted.  Returns pipe.finish().
int submit_flagged(FilePipeline& pipe, const std::vector<swec_damage_range>& runs, size_t chunk, const std::vector<int>& in,
                   const std::vector<int>& in_d, const std::function<void(Item&)>& add) {
    std::vector<std::pair<int64_t, int64_t>> spans;
    for (const swec_damage_range& r : runs) spans.push_back({r.offset, r.offset + r.length});
    std::sort(spans.begin(), spans.end());
    size_t nspans = 0;
    for (const auto& sp : spans) {
        if (nspans && sp.first <= spans[nspans - 1].second) spans[nspans - 1].second = std::max(spans[nspans - 1].second, sp.second);
        else spans[nspans++] = sp;
    }
    spans.resize(nspans);
    int rc = SWEC_OK;
    for (size_t sp = 0; rc == SWEC_OK && sp < spans.size(); sp++)
        for (int64_t o = spans[sp].first; rc == SWEC_OK && o < spans[sp].second; o += int64_t(chunk)) {
            Item it;
            it.len = size_t(std::min<int64_t>(int64_t(chunk), spans[sp].second - o));
            it.shard_off = o;
            for (size_t i = 0; i < in.size(); i++) it.reads.push_back({int(i), in[i], o, 0, it.len, in_d[i]});
            if (add) add(it);
            rc = pipe.submit(std::move(it));
        }
    return pipe.finish();
}

// The writes of the repairs' pass 2: each blamed shard gets back only its own pages of pass 1's `runs`, through out[i]
// (out_d[i]: its O_DIRECT twin, -1 = none), which the caller opens for the blamed shards alone.
class PageWrites {
  public:
    std::vector<int> out, out_d;

    PageWrites(const std::vector<swec_damage_range>& runs, int total)
        : out(size_t(total), -1), out_d(size_t(total), -1), runs_(runs), next_(size_t(total), 0), stop_(size_t(total), 0) {
        // each shard's slice of `runs`, which lists them shard by shard in ascending offset; an empty one: not blamed
        for (size_t r = runs.size(); r-- > 0;)
            if (runs[r].shard_id >= 0) {
                const size_t id = size_t(runs[r].shard_id);
                if (!stop_[id]) stop_[id] = r + 1;
                next_[id] = r;
            }
    }
    bool blamed(int i) const { return stop_[size_t(i)] > 0; }

    // the writes of the next item, which submit_flagged hands over in ascending shard offset
    void add(Item& it) {
        const int64_t o = it.shard_off, end = o + int64_t(it.len);
        for (size_t i = 0; i < out.size(); i++)
            for (size_t& r = next_[i]; r < stop_[i]; r++) {  // shard i's own pages in the item
                const int64_t lo = std::max(runs_[r].offset, o), hi = std::min(runs_[r].offset + runs_[r].length, end);
                if (lo >= end) break;
                it.writes.push_back({int(i), out[i], lo, size_t(lo - o), size_t(hi - lo), out_d[i]});
                if (hi < runs_[r].offset + runs_[r].length) break;  // the run goes on in the next item
            }
    }

    // every modified file made durable; `base` + the shard's extension names a failing one
    int sync(const std::string& base) const {
        for (size_t i = 0; i < out.size(); i++)
            if (out[i] >= 0 && fdatasync(out[i]) != 0) return io_fail("fdatasync " + base + shard_ext(int(i)));
        return SWEC_OK;
    }

  private:
    const std::vector<swec_damage_range>& runs_;
    std::vector<size_t> next_, stop_;
};

// Pass 2 of swec_repair_ec_damage.  `runs` are every page run pass 1 found, of the blamed shards and of the
// uncorrectable columns.  Only the columns of those pages go through the pipeline again, with a correcting locator, and
// the report and ranges are collected from that.  Each blamed shard gets back only its own pages, in the file where it
// was found, made durable before the call returns.
int repair_pages(swec_encoder* enc, const Matrix& rows, const std::string& b, const char* const* dirs, int ndirs,
                 const std::vector<int>& in, int64_t size, int radius, const std::vector<swec_damage_range>& runs,
                 swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges) {
    const int total = int(in.size());
    PageWrites writes(runs, total);
    FdSet fds;
    const long direct = g_opt_file_direct_io.load();
    std::vector<int> in_d(static_cast<size_t>(total), -1);
    for (int i = 0; i < total; i++) {
        const std::string path = find_shard_file(b, dirs, ndirs, i);
        in_d[size_t(i)] = fds.keep(open_direct(path, O_RDONLY, direct & 1));
        if (!writes.blamed(i)) continue;
        if ((writes.out[size_t(i)] = fds.keep(open(path.c_str(), O_RDWR))) < 0) return io_fail("open " + path);
        writes.out_d[size_t(i)] = fds.keep(open_direct(path, O_RDWR, direct & 2));
    }
    const size_t chunk = file_chunk(size);
    DamageLocator locator;
    FilePipeline pipe(enc, rows, chunk, rows.rows, locate_step(locator));
    int rc = pipe.start();
    if (rc) return rc;
    if ((rc = locator.init(rows, size, radius, enc->stream, /*correct=*/true))) return rc;
    if ((rc = submit_flagged(pipe, runs, chunk, in, in_d, [&](Item& it) { writes.add(it); }))) return rc;
    pipe.report("repair_ec_damage");
    if ((rc = writes.sync(b))) return rc;
    return locator.collect(report, ranges, ranges_cap, n_ranges);
}

// Pass 1 of the damage calls, swec_locate_ec_damage itself: every column of the k+m shard files `in`, all `size` bytes,
// through a pipeline that reads the m parity shards too and runs the locator on each slot.  `runs` (may be NULL)
// receives every page run, for pass 2.
int locate_pass(swec_encoder* enc, const Matrix& rows, const std::vector<int>& in, int64_t size, int radius,
                swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges,
                std::vector<swec_damage_range>* runs) {
    const size_t chunk = file_chunk(size);
    DamageLocator locator;
    FilePipeline pipe(enc, rows, chunk, rows.rows, locate_step(locator));
    int rc = pipe.start();
    if (rc) return rc;
    rc = locator.init(rows, size, radius, enc->stream);
    if (rc == SWEC_OK) rc = scrub_columns(pipe, in, size, chunk);
    if (rc == SWEC_OK) rc = locator.collect(report, ranges, ranges_cap, n_ranges, runs);
    return rc;
}  // the pipeline parks its staging ring for pass 2

// swec_locate_ec_damage, and with `repair` swec_repair_ec_damage, whose pass 1 is the locate call itself: a set without
// damage is never opened for writing.
int damage_files(const char* base, const char* const* dirs, int ndirs, int k, int m, int device, int radius, bool repair,
                 swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges, int* ok) {
    if (!base || !ok || (ndirs > 0 && !dirs)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    *ok = 0;
    const std::string b(base);
    if (k == 0) ec_ratio(b, &k, &m);
    int rc = check_locate_args(m, radius, report, ranges, ranges_cap);
    if (rc) return rc;
    CallEncoder enc;
    if ((rc = new_call_encoder(k, m, device, &enc))) return rc;
    FdSet fds;
    std::vector<int> in;
    int64_t size = -1;
    if ((rc = open_all_shards(b, dirs, ndirs, k + m, &fds, &in, &size))) return rc;
    const Matrix rows = parity_rows(enc.get());
    std::vector<swec_damage_range> runs;
    if ((rc = locate_pass(enc.get(), rows, in, size, radius, report, ranges, ranges_cap, n_ranges, repair ? &runs : nullptr)))
        return rc;
    if (repair && report->damaged_columns &&
        (rc = repair_pages(enc.get(), rows, b, dirs, ndirs, in, size, radius, runs, report, ranges, ranges_cap, n_ranges)))
        return rc;
    *ok = (repair ? report->uncorrectable_columns : report->damaged_columns) == 0 ? 1 : 0;
    return SWEC_OK;
}

// What the checked rebuild adds to swec_rebuild_ec_files: the radius and where the report goes.
struct Checked {
    int radius;
    swec_damage_report* report;
    swec_damage_range* ranges;
    int ranges_cap;
    int* n_ranges;
    bool checked = false;  // set once the report comes from a locator (c >= 1)
};

// Submits an item whose length is set, at shard offset `col`: the caller adds what else the item needs.
using SubmitFn = std::function<int(Item&& it, int64_t col)>;
// Adds what an item needs of one stripe row segment: columns [col, col + len) of the row whose k blocks start at .dat
// offset row_dat, `block` bytes apart (`tail`: the last, partial small row), at offset src of the item's streams.
using RowFn = std::function<void(Item& it, int64_t row_dat, int64_t block, bool tail, int64_t col, int64_t len, size_t src)>;

// The items of a .dat's striping (ec_encoder.go:280-321), in order: rows of large blocks cut at the slot size, then the
// small rows, chunk / small to an item (row by row, cut at the slot size, when a small block is bigger than a slot),
// the tail row last and `tail_width` columns wide.  No item straddles a row of large blocks.  Every row segment of an
// item goes to row(), then the item to submit(); the walk stops at the first failed submit and returns its status.
int walk_items(const StripeGeometry& g, size_t chunk, int64_t tail_width, const RowFn& row, const SubmitFn& submit) {
    int rc = SWEC_OK;
    const auto cut = [&](int64_t row_dat, int64_t block, bool tail, int64_t width, int64_t col0) {
        for (int64_t o = 0; rc == SWEC_OK && o < width; o += int64_t(chunk)) {
            Item it;
            it.len = size_t(std::min<int64_t>(int64_t(chunk), width - o));
            row(it, row_dat, block, tail, o, int64_t(it.len), 0);
            rc = submit(std::move(it), col0 + o);
        }
    };
    for (int64_t r = 0; r < g.large_rows; r++) cut(r * g.large_row(), g.large, false, g.large, r * g.large);
    const int64_t nrows = g.small_rows + (g.tail > 0 ? 1 : 0);
    const auto width = [&](int64_t j) { return j < g.small_rows ? g.small : tail_width; };
    const auto row_dat = [&](int64_t j) { return g.small_dat_offset() + j * g.small_row(); };
    const auto col = [&](int64_t j) { return g.small_shard_offset() + j * g.small; };
    if (g.small > int64_t(chunk)) {
        for (int64_t j = 0; j < nrows; j++) cut(row_dat(j), g.small, j == g.small_rows, width(j), col(j));
        return rc;
    }
    // Small rows are tiny (10 x 1 MiB): many of them share one slot.  Row j of an item scatters to offset j * small of
    // its streams, so every shard still takes ONE contiguous run per item.  A default 30,000 MiB volume is 2 large
    // rows + 952 small ones: a third of its bytes take this path.
    const int64_t rows_per_item = int64_t(chunk) / g.small;
    for (int64_t first = 0; rc == SWEC_OK && first < nrows; first += rows_per_item) {
        Item it;
        for (int64_t j = first; j < std::min(nrows, first + rows_per_item); j++) {
            row(it, row_dat(j), g.small, j == g.small_rows, 0, width(j), it.len);
            it.len += size_t(width(j));
        }
        rc = submit(std::move(it), col(first));
    }
    return rc;
}

// The pipeline of the checked rebuild and decode over columns [0, cols) of the shards, after reserving `reserve_size`
// bytes of each file in `reserve`.  The items `walk` gives, in slots of `chunk` columns, each read the k information
// and c check streams at their plan positions.  Per slot: one apply of plan.fused (the check shards re-encoded, the
// missing shards rebuilt), then, with c >= 1, the rebuilding or decoding locator, which compares the c check rows with
// the stored ones and corrects the errors it locates in the information set.  With c = 0 (exactly k shards present)
// the set is rebuilt and the report says nothing was checked.
int checked_pipeline(swec_encoder* enc, const CheckedPlan& plan, const std::vector<int>& in, const std::vector<int>& in_d,
                     int64_t cols, const std::vector<int>& reserve, int64_t reserve_size, Checked* chk,
                     const std::function<int(size_t chunk, const SubmitFn& submit)>& walk) {
    const int k = enc->k, c = plan.c();
    const size_t chunk = file_chunk(cols);
    DamageLocator locator;
    FilePipeline pipe(enc, plan.fused, chunk, c, c > 0 ? locate_step(locator) : FilePipeline::Step{});
    int rc = pipe.start();
    if (rc) return rc;
    if (c > 0 && (rc = locator.init_rebuild(plan, cols, chk->radius, enc->stream))) return rc;
    if (!reserve.empty()) reserve_extents(reserve, reserve_size);
    walk(chunk, [&](Item&& it, int64_t col) {
        it.shard_off = col;
        for (int p = 0; p < k + c; p++) {
            const size_t id = size_t(p < k ? plan.info[size_t(p)] : plan.check(p - k));
            it.reads.push_back({p, in[id], col, 0, it.len, in_d[id]});
        }
        return pipe.submit(std::move(it));
    });  // a failed submit ends the walk, and finish() returns its error
    if ((rc = pipe.finish())) return rc;
    if (c == 0) {
        unchecked_report(chk->report, chk->n_ranges);
        return SWEC_OK;
    }
    if ((rc = locator.collect(chk->report, chk->ranges, chk->ranges_cap, chk->n_ranges))) return rc;
    chk->checked = true;
    return SWEC_OK;
}

// The checked rebuild: every present shard is read, as the check shards of the punctured code beyond the first k, and
// the rebuilt shards are written to `out` (in ascending id of the missing shards).
int rebuild_checked(swec_encoder* enc, const std::vector<int>& in, const std::vector<int>& in_d,
                    const std::vector<uint8_t>& present, const std::vector<int>& out, const std::vector<int>& out_d,
                    int64_t todo, Checked* chk) {
    CheckedPlan plan;
    if (!plan.build(enc->gen, enc->k, present.data(), /*decode=*/false)) return fail(SWEC_ERR_TOO_FEW_SHARDS, "not enough shards");
    return checked_pipeline(enc, plan, in, in_d, todo, out, todo, chk, [&](size_t chunk, const SubmitFn& submit) {
        int rc = SWEC_OK;
        for (int64_t o = 0; rc == SWEC_OK && o < todo; o += int64_t(chunk)) {
            Item it;
            it.len = size_t(std::min<int64_t>(int64_t(chunk), todo - o));
            for (size_t r = 0; r < out.size(); r++)
                it.writes.push_back({plan.position(plan.rebuilt(int(r))), out[r], o, 0, it.len, out_d[r]});
            rc = submit(std::move(it), o);
        }
        return rc;
    });
}

// swec_rebuild_ec_files, and with `chk` swec_rebuild_ec_files_checked: the same files, checks, errors and order.  The
// checked rebuild reads every present shard, not only the first k, and corrects the damage it locates in the first k
// before it reaches the rebuilt shards.
int rebuild_files(const char* base, const char* const* dirs, int ndirs, int k, int m, int device, uint32_t* rebuilt,
                  int* n_rebuilt, Checked* chk) {
    if (!base || !rebuilt || !n_rebuilt || (ndirs > 0 && !dirs)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    *n_rebuilt = 0;
    const std::string b(base);
    if (k == 0) ec_ratio(b, &k, &m);  // RebuildEcFiles (ec_encoder.go:76-95)
    CallEncoder enc;
    int rc = new_call_encoder(k, m, device, &enc);
    if (rc) return rc;
    const int total = k + m;

    // pass 1: which shards exist
    FdSet fds;
    const long direct = g_opt_file_direct_io.load();
    std::vector<int> in(static_cast<size_t>(total), -1), in_d(static_cast<size_t>(total), -1);
    std::vector<uint8_t> present(static_cast<size_t>(total), 0);
    std::vector<uint32_t> missing;
    for (int i = 0; i < total; i++) {
        if ((rc = open_shard(b, dirs, ndirs, i, &fds, &in[size_t(i)], &in_d[size_t(i)], direct & 1))) return rc;
        present[size_t(i)] = in[size_t(i)] >= 0;
        if (!present[size_t(i)]) missing.push_back(uint32_t(i));
    }
    const int npresent = total - int(missing.size());
    if (npresent < k)  // before any output file exists — ec_encoder.go:172-175
        return fail(SWEC_ERR_TOO_FEW_SHARDS, "not enough shards to rebuild " + b + ": found " + std::to_string(npresent) +
                                                 " shards, need at least " + std::to_string(k));
    for (uint32_t id : missing) rebuilt[(*n_rebuilt)++] = id;
    if (missing.empty() && !chk) return SWEC_OK;  // the checked call still checks the set

    // pass 2: create the outputs — ec_encoder.go:182-193.  Whatever goes wrong from here on, the caller gets no
    // shard ids (the reference returns nil ids with the error) and no half-written output survives: a shard file
    // that exists is taken for a present input by the next rebuild (findShardFile), so a partial one must not stay.
    std::vector<int> out, out_d;  // in the order of `missing`
    struct Undo {
        const std::string& b;
        const std::vector<uint32_t>& ids;
        int* n_rebuilt;
        size_t created = 0;
        bool armed = true;
        ~Undo() {
            if (!armed) return;
            for (size_t i = 0; i < created; i++) unlink((b + shard_ext(int(ids[i]))).c_str());
            *n_rebuilt = 0;
        }
    } undo{b, missing, n_rebuilt};
    for (uint32_t id : missing) {
        const int fd = fds.keep(open((b + shard_ext(int(id))).c_str(), O_TRUNC | O_WRONLY | O_CREAT, 0644));
        if (fd < 0) return io_fail("create " + b + shard_ext(int(id)));
        undo.created++;
        out.push_back(fd);
        out_d.push_back(fds.keep(open_direct(b + shard_ext(int(id)), O_WRONLY, direct & 2)));
    }

    // every present shard must have the same length; the reference steps in 1 MiB reads and fails at the first
    // short, unequal one
    int64_t size = -1;
    for (int fd : in)
        if (fd >= 0 && (rc = check_length(fd, &size))) return rc;
    // quirk kept: the reference reads in small-block buffers, and a length above 1 MiB that is not a multiple of
    // 1 MiB errors on the last read
    const int64_t mib = kSmallBlockSize;
    const bool ragged = !missing.empty() && size > mib && size % mib != 0;
    const int64_t todo = ragged ? size / mib * mib : size;

    if (chk) {
        if ((rc = rebuild_checked(enc.get(), in, in_d, present, out, out_d, todo, chk))) return rc;
    } else {
        std::vector<int> ins, outs_idx;  // outs_idx == missing: fused row r rebuilds the shard of out[r]
        Matrix fused;
        if (!rs_reconstruct_plan(enc->gen, k, present.data(), false, &ins, &outs_idx, &fused))
            return fail(SWEC_ERR_TOO_FEW_SHARDS, "not enough shards");
        const size_t chunk = file_chunk(todo);
        FilePipeline pipe(enc.get(), fused, chunk);
        if ((rc = pipe.start())) return rc;
        reserve_extents(out, todo);
        for (int64_t o = 0; rc == SWEC_OK && o < todo; o += int64_t(chunk)) {
            Item it;
            it.len = size_t(std::min<int64_t>(int64_t(chunk), todo - o));
            for (int i = 0; i < k; i++) it.reads.push_back({i, in[size_t(ins[size_t(i)])], o, 0, it.len, in_d[size_t(ins[size_t(i)])]});
            for (size_t r = 0; r < out.size(); r++) it.writes.push_back({k + int(r), out[r], o, 0, it.len, out_d[r]});
            rc = pipe.submit(std::move(it));
        }
        if ((rc = pipe.finish())) return rc;
    }
    if (ragged) return shard_size_error(mib, size % mib);
    undo.armed = false;
    return SWEC_OK;
}

// The checked decode over columns [0, cols) of the shards, in the items of walk_items() with the tail row as wide as
// shard 0's part of it.  The apply computes the rows of the missing data shards and of the check shards, and the
// decoding locator also corrects the information streams that are data shards in the slot.  The item's writes un-stripe
// the k data streams into the .dat at the plan's offsets; shard s holds tail_bytes(s) of the tail row.
int decode_dat(swec_encoder* enc, const std::vector<int>& in, const std::vector<int>& in_d,
               const std::vector<uint8_t>& present, int dat, int dat_d, const StripeGeometry& g, int64_t dat_size,
               int64_t cols, Checked* chk) {
    const int k = enc->k;
    CheckedPlan plan;
    if (!plan.build(enc->gen, k, present.data(), /*decode=*/true)) return fail(SWEC_ERR_TOO_FEW_SHARDS, "not enough shards");
    std::vector<int> stream(static_cast<size_t>(k));  // the slot stream that holds data shard s
    for (int s = 0; s < k; s++) stream[size_t(s)] = plan.position(s);
    const RowFn unstripe = [&](Item& it, int64_t row_dat, int64_t block, bool tail, int64_t col, int64_t len, size_t src) {
        for (int s = 0; s < k; s++) {
            const int64_t n = std::min(len, (tail ? g.tail_bytes(s) : block) - col);
            if (n > 0) it.writes.push_back({stream[size_t(s)], dat, row_dat + int64_t(s) * block + col, src, size_t(n), dat_d});
        }
    };
    return checked_pipeline(enc, plan, in, in_d, cols, {dat}, dat_size, chk, [&](size_t chunk, const SubmitFn& submit) {
        return walk_items(g, chunk, g.tail_bytes(0), unstripe, submit);
    });
}

}  // namespace

namespace swec {

// Pass 2 per item: the slot's data shards saved, the correcting locate, the corrected data re-encoded into the computed
// rows (the locate is done with them), then the attribution.  Without `repair` nothing comes back to the host and
// nothing is written.  With it, the writes of swec_repair_ec_damage's pass 2 go to the inodes behind `in`: each blamed
// shard's descriptor is opened again for writing through /proc/self/fd before anything is read again, and the call
// fails there, with nothing written, when that is refused.
int needle_damage_files(swec_encoder* enc, const std::vector<int>& in, int64_t size, int radius, const StripeMap& map,
                        int version, bool repair, std::vector<swec_needle_damage>* recs, swec_damage_report* report,
                        swec_damage_range* ranges, int ranges_cap, int* n_ranges, uint64_t unowned[2]) {
    const Matrix rows = parity_rows(enc);
    std::vector<swec_damage_range> runs;
    int rc = locate_pass(enc, rows, in, size, radius, report, ranges, ranges_cap, n_ranges, &runs);
    if (rc || report->damaged_columns == 0) return rc;
    const int k = enc->k;
    PageWrites writes(runs, int(in.size()));
    FdSet fds;
    const long direct = g_opt_file_direct_io.load();
    for (int i = 0; repair && i < int(in.size()); i++) {
        if (!writes.blamed(i)) continue;
        const std::string self = "/proc/self/fd/" + std::to_string(in[size_t(i)]);
        if ((writes.out[size_t(i)] = fds.keep(open(self.c_str(), O_RDWR))) < 0)
            return io_fail("open shard " + shard_ext(i) + " for writing through " + self);
        writes.out_d[size_t(i)] = fds.keep(open_direct(self, O_RDWR, direct & 2));
    }
    const size_t chunk = file_chunk(size);
    DamageLocator locator;
    NeedleDamage nd;
    FilePipeline pipe(enc, rows, chunk, rows.rows, [&](uint8_t* const* computed, uint8_t* const* shards, size_t len,
                                                      int64_t base, int slot, cudaStream_t s) -> int {
        int r = nd.save(shards, len, slot, s);
        if (r == SWEC_OK) r = locator.launch(computed, shards, len, base, s);
        if (r == SWEC_OK) {
            const uint8_t* data[SWEC_MAX_SHARDS];
            for (int i = 0; i < k; i++) data[i] = shards[i];
            std::lock_guard<std::mutex> lk(enc->mu);
            r = enc->apply(rows, data, computed, len, Layout{}, s);
        }
        if (r == SWEC_OK) r = nd.launch(nullptr, shards, computed, len, base, slot, s);
        return r;
    });
    if ((rc = pipe.start())) return rc;
    if ((rc = locator.init(rows, size, radius, enc->stream, /*correct=*/true))) return rc;
    if ((rc = nd.init(k, enc->m, map, recs->data(), int(recs->size()), version, int(pipe.slot_count()), chunk, enc->stream)))
        return rc;
    const std::function<void(Item&)> add = [&](Item& it) { writes.add(it); };
    if ((rc = submit_flagged(pipe, runs, chunk, in, std::vector<int>(in.size(), -1), repair ? add : nullptr))) return rc;
    pipe.report(repair ? "repair_needle_damage" : "locate_needle_damage");
    if ((rc = writes.sync(""))) return rc;
    return nd.collect(recs->data(), unowned);
}

}  // namespace swec

extern "C" {

int swec_generate_ec_files(const char* base, int64_t buffer_size, int64_t large, int64_t small, int k, int m,
                           int device) {
    if (!base) return fail(SWEC_ERR_INVALID_ARG, "base_file_name is NULL");
    const double t_call = PipeStats::now();
    // encodeData: "unexpected zero buffer size" / "unexpected block size %d buffer size %d" (ec_encoder.go:204-212)
    if (buffer_size <= 0 || large <= 0 || small <= 0 || large % buffer_size || small % buffer_size)
        return fail(SWEC_ERR_INVALID_ARG, "block sizes must be positive multiples of buffer_size");
    CallEncoder enc;
    int rc = new_call_encoder(k, m, device, &enc);
    if (rc) return rc;

    const std::string b(base);
    FdSet fds;
    const int dat = fds.keep(open((b + ".dat").c_str(), O_RDONLY));
    if (dat < 0) return io_fail("failed to open dat file " + b + ".dat");
    struct stat st;
    if (fstat(dat, &st) != 0) return io_fail("failed to stat dat file");
    const int total = k + m;
    const long direct = g_opt_file_direct_io.load();
    const int dat_d = fds.keep(open_direct(b + ".dat", O_RDONLY, direct & 1));
    std::vector<int> outs(static_cast<size_t>(total), -1), outs_d(static_cast<size_t>(total), -1);
    {
        // openEcFiles (ec_encoder.go:224-238): O_TRUNC|O_CREAT|O_WRONLY 0644 for every shard — all at once.  Truncating
        // a shard file left by an earlier encode frees its pages one file after the other when done in a loop: 2.2 s
        // for the 11 GiB of shards of an 8 GiB volume on tmpfs, several times the encode itself.
        std::vector<int> err(static_cast<size_t>(total), 0);
        std::vector<std::thread> openers;
        for (int i = 0; i < total; i++)
            openers.emplace_back([&, i] {
                outs[size_t(i)] = open((b + shard_ext(i)).c_str(), O_TRUNC | O_CREAT | O_WRONLY, 0644);
                if (outs[size_t(i)] < 0) err[size_t(i)] = errno;
                else outs_d[size_t(i)] = open_direct(b + shard_ext(i), O_WRONLY, direct & 2);
            });
        for (auto& t : openers) t.join();
        for (int i = 0; i < total; i++) {
            fds.keep(outs[size_t(i)]);
            fds.keep(outs_d[size_t(i)]);
        }
        for (int i = 0; i < total; i++)
            if (outs[size_t(i)] < 0) {
                errno = err[size_t(i)];
                return io_fail("failed to open file " + b + shard_ext(i));
            }
    }

    const Matrix rows = parity_rows(enc.get());
    const size_t chunk = file_chunk(std::max(large, small));
    const double t_opened = PipeStats::now();
    FilePipeline pipe(enc.get(), rows, chunk);
    if ((rc = pipe.start())) return rc;
    const StripeGeometry g(st.st_size, k, large, small);
    pipe.stats.prealloc += reserve_extents(outs, g.shard_size());

    // encodeData (ec_encoder.go:304-319): the tail row is read as a whole small row, zero past EOF (ec_encoder.go:258-262)
    walk_items(
        g, chunk, small,
        [&](Item& it, int64_t row_dat, int64_t block, bool, int64_t col, int64_t len, size_t src) {
            for (int i = 0; i < k; i++) it.reads.push_back({i, dat, row_dat + block * i + col, src, size_t(len), dat_d});
        },
        [&](Item&& it, int64_t col) {
            for (int i = 0; i < total; i++) it.writes.push_back({i, outs[size_t(i)], col, 0, it.len, outs_d[size_t(i)]});
            return pipe.submit(std::move(it));
        });
    rc = pipe.finish();  // the first error, submit()'s included
    pipe.report("generate_ec_files");
    const double t_piped = PipeStats::now();
    pipe.shutdown();
    if (getenv("SWEC_PIPE_STATS"))
        fprintf(stderr, "{\"call\": \"generate_ec_files\", \"dat_bytes\": %lld, \"open_and_truncate_s\": %.3f, \"pipeline_s\": %.3f, "
                        "\"teardown_s\": %.3f}\n",
                (long long)st.st_size, t_opened - t_call, t_piped - t_opened, PipeStats::now() - t_piped);
    return rc;
}

int swec_write_ec_files(const char* base, int device) {
    return swec_generate_ec_files(base, kBufferSize, kLargeBlockSize, kSmallBlockSize, kDefaultDataShards,
                                  kDefaultParityShards, device);
}

int swec_rebuild_ec_files(const char* base, const char* const* dirs, int ndirs, int k, int m, int device,
                          uint32_t* rebuilt, int* n_rebuilt) {
    return rebuild_files(base, dirs, ndirs, k, m, device, rebuilt, n_rebuilt, nullptr);
}

int swec_rebuild_ec_files_checked(const char* base, const char* const* dirs, int ndirs, int k, int m, int device,
                                  int radius, uint32_t* rebuilt, int* n_rebuilt, swec_damage_report* report,
                                  swec_damage_range* ranges, int ranges_cap, int* n_ranges, int* ok) {
    if (!base || !rebuilt || !n_rebuilt || !ok || (ndirs > 0 && !dirs)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    *ok = 0;
    *n_rebuilt = 0;
    if (const int rc = check_rebuild_args(radius, report, ranges, ranges_cap)) return rc;
    Checked chk{radius, report, ranges, ranges_cap, n_ranges};
    const int rc = rebuild_files(base, dirs, ndirs, k, m, device, rebuilt, n_rebuilt, &chk);
    *ok = rc == SWEC_OK && chk.checked && report->uncorrectable_columns == 0 ? 1 : 0;
    return rc;
}

int swec_verify_ec_files(const char* base, const char* const* dirs, int ndirs, int k, int m, int device,
                         uint64_t* mismatched_vectors, int* ok) {
    if (!base || !ok || (ndirs > 0 && !dirs)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    *ok = 0;
    const std::string b(base);
    if (k == 0) ec_ratio(b, &k, &m);
    CallEncoder enc;
    int rc = new_call_encoder(k, m, device, &enc);
    if (rc) return rc;
    FdSet fds;
    std::vector<int> in;
    int64_t size = -1;
    if ((rc = open_all_shards(b, dirs, ndirs, k + m, &fds, &in, &size))) return rc;
    const Matrix rows = parity_rows(enc.get());
    const size_t chunk = file_chunk(size);
    // mismatching 16-byte vectors per parity row, zeroed before any slot stream compares into them; declared before
    // the pipeline so that they are freed only after its shutdown has drained every compare
    if ((rc = enc->ensure_device())) return rc;
    StreamScratch dev_bad(enc->stream);
    const size_t bad_bytes = sizeof(unsigned long long) * size_t(m);
    SWEC_CUDA(dev_bad.alloc(bad_bytes));
    SWEC_CUDA(cudaMemsetAsync(dev_bad.p, 0, bad_bytes, enc->stream));
    SWEC_CUDA(cudaStreamSynchronize(enc->stream));
    FilePipeline pipe(enc.get(), rows, chunk, m, [&](uint8_t* const* computed, uint8_t* const* shards, size_t len, int64_t,
                                                     int, cudaStream_t s) -> int {
        for (int r = 0; r < m; r++) SWEC_CUDA(launch_compare(computed[r], shards[k + r], len, dev_bad.as<unsigned long long>() + r, s));
        return SWEC_OK;
    });
    if ((rc = pipe.start())) return rc;
    std::vector<unsigned long long> bad(static_cast<size_t>(m), 0);
    if ((rc = scrub_columns(pipe, in, size, chunk))) return rc;
    SWEC_CUDA(cudaMemcpy(bad.data(), dev_bad.p, bad_bytes, cudaMemcpyDeviceToHost));
    bool all_ok = true;
    for (int p = 0; p < m; p++) {
        if (mismatched_vectors) mismatched_vectors[p] = bad[size_t(p)];
        all_ok = all_ok && bad[size_t(p)] == 0;
    }
    *ok = all_ok ? 1 : 0;
    return SWEC_OK;
}

int swec_locate_ec_damage(const char* base, const char* const* dirs, int ndirs, int k, int m, int device, int radius,
                          swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges, int* ok) {
    return damage_files(base, dirs, ndirs, k, m, device, radius, false, report, ranges, ranges_cap, n_ranges, ok);
}

int swec_repair_ec_damage(const char* base, const char* const* dirs, int ndirs, int k, int m, int device, int radius,
                          swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges, int* ok) {
    return damage_files(base, dirs, ndirs, k, m, device, radius, true, report, ranges, ranges_cap, n_ranges, ok);
}

int swec_write_dat_file(const char* base, int64_t dat_size, const char* const* shard_names, int k, int64_t large,
                        int64_t small) {
    if (!base || !shard_names || k <= 0 || k > SWEC_MAX_SHARDS || large <= 0 || small <= 0 || dat_size < 0)
        return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    FdSet fds;
    const int dat = fds.keep(open((std::string(base) + ".dat").c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644));
    if (dat < 0) return io_fail("cannot write volume .dat");
    std::vector<int> in;
    for (int i = 0; i < k; i++) {
        in.push_back(fds.keep(open(shard_names[i], O_RDONLY)));
        if (in.back() < 0) return io_fail(std::string("open ") + shard_names[i]);
    }
    // The copy plan of the reference's two loops (ec_decoder.go:200-219) — shard s is read sequentially, the .dat is
    // written sequentially — as independent (shard offset → .dat offset) pieces, executed in parallel: every piece
    // has explicit offsets on both sides, so the order of execution cannot change the bytes.
    struct Piece { int shard; int64_t shard_off, dat_off, len; };
    std::vector<Piece> pieces;
    const int64_t max_piece = int64_t(8) << 20;
    std::vector<int64_t> pos(static_cast<size_t>(k), 0);
    int64_t out = 0;
    auto plan = [&](int shard, int64_t n) {  // io.CopyN(datFile, inputFiles[shard], n)
        for (int64_t o = 0; o < n; o += max_piece)
            pieces.push_back({shard, pos[size_t(shard)] + o, out + o, std::min(max_piece, n - o)});
        pos[size_t(shard)] += n;
        out += n;
    };
    const StripeGeometry g(dat_size, k, large, small);
    for (int64_t r = 0; r < g.large_rows; r++)
        for (int s = 0; s < k; s++) plan(s, large);
    for (int64_t r = 0; r < g.small_rows; r++)
        for (int s = 0; s < k; s++) plan(s, small);
    for (int s = 0; s < k; s++)  // the last row: min(remaining, small) each; shards past the end get nothing
        if (const int64_t n = g.tail_bytes(s)) plan(s, n);
    // a shard shorter than the plan needs is the reference's "copy … block" error: check before writing anything
    for (int s2 = 0; s2 < k; s2++) {
        struct stat st;
        if (fstat(in[size_t(s2)], &st) != 0) return io_fail("fstat shard");
        if (st.st_size < pos[size_t(s2)]) return fail(SWEC_ERR_IO, "short read copying shard " + std::to_string(s2));
    }
    if (ftruncate(dat, off_t(dat_size)) != 0) return io_fail("size .dat");
    FirstError first;
    const std::function<int(int)> copy_piece = [&](int idx) -> int {
        const Piece& pc = pieces[size_t(idx)];
        int64_t done = 0;
        // kernel-side copy first (no user-space bounce; shares extents where the filesystem can) …
        while (done < pc.len) {
            off64_t oi = pc.shard_off + done, oo = pc.dat_off + done;
            const ssize_t n = copy_file_range(in[size_t(pc.shard)], &oi, dat, &oo, size_t(pc.len - done), 0);
            if (n <= 0) break;  // unsupported combination, or EOF: the read/write loop below decides
            done += n;
        }
        // … plain pread/pwrite for whatever is left
        std::vector<uint8_t> buf;
        while (done < pc.len) {
            if (buf.empty()) buf.resize(size_t(std::min<int64_t>(pc.len, int64_t(4) << 20)));
            const size_t want = size_t(std::min<int64_t>(pc.len - done, int64_t(buf.size())));
            const ssize_t got = pread(in[size_t(pc.shard)], buf.data(), want, off_t(pc.shard_off + done));
            if (got < 0 && errno == EINTR) continue;
            if (got <= 0) return first.fail(SWEC_ERR_IO, "short read copying shard " + std::to_string(pc.shard));
            ssize_t put = 0;
            while (put < got) {
                const ssize_t w = pwrite(dat, buf.data() + put, size_t(got - put), off_t(pc.dat_off + done + put));
                if (w < 0 && errno == EINTR) continue;
                if (w <= 0) return first.fail(SWEC_ERR_IO, std::string("write .dat: ") + strerror(errno));
                put += w;
            }
            done += got;
        }
        return SWEC_OK;
    };
    return file_io_pool().parallel_for(int(pieces.size()), copy_piece) ? first.get() : SWEC_OK;
}


int swec_write_dat_file_checked(const char* base, int64_t dat_size, const char* const* names, int k, int m, int64_t large,
                                int64_t small, int device, int radius, swec_damage_report* report,
                                swec_damage_range* ranges, int ranges_cap, int* n_ranges, int* ok) {
    if (!base || !names || !ok || k <= 0 || m <= 0 || k + m > SWEC_MAX_SHARDS || large <= 0 || small <= 0 || dat_size < 0)
        return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    *ok = 0;
    int rc = check_rebuild_args(radius, report, ranges, ranges_cap);
    if (rc) return rc;
    const int total = k + m;
    FdSet fds;
    const long direct = g_opt_file_direct_io.load();
    std::vector<int> in(static_cast<size_t>(total), -1), in_d(static_cast<size_t>(total), -1);
    std::vector<uint8_t> present(static_cast<size_t>(total), 0);
    int npresent = 0;
    for (int i = 0; i < total; i++) {
        if (!names[i]) continue;
        if ((in[size_t(i)] = fds.keep(open(names[i], O_RDONLY))) < 0) return io_fail(std::string("open ") + names[i]);
        in_d[size_t(i)] = fds.keep(open_direct(names[i], O_RDONLY, direct & 1));
        present[size_t(i)] = 1;
        npresent++;
    }
    // every check before the .dat exists: enough shards, of one length, long enough for the copy plan
    if (npresent < k)
        return fail(SWEC_ERR_TOO_FEW_SHARDS, "not enough shards to decode " + std::string(base) + ": found " +
                                                 std::to_string(npresent) + " shards, need at least " + std::to_string(k));
    int64_t size = -1;
    for (int fd : in)
        if (fd >= 0 && (rc = check_length(fd, &size))) return rc;
    const StripeGeometry g(dat_size, k, large, small);
    for (int s = 0; s < k; s++)  // what the plan reads from shard s (ec_decoder.go:200-219); shard 0 reads the most
        if (size < g.tail_shard_offset() + g.tail_bytes(s)) return fail(SWEC_ERR_IO, "short read copying shard " + std::to_string(s));
    bool all_data = true;
    for (int s = 0; s < k; s++) all_data = all_data && present[size_t(s)];
    if (all_data && npresent == k) {  // the data shards alone: nothing to check, nothing to rebuild
        unchecked_report(report, n_ranges);
        return swec_write_dat_file(base, dat_size, names, k, large, small);
    }
    CallEncoder enc;
    if ((rc = new_call_encoder(k, m, device, &enc))) return rc;
    const std::string path = std::string(base) + ".dat";
    const int dat = fds.keep(open(path.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644));
    if (dat < 0) return io_fail("cannot write volume .dat");
    struct Undo {  // only a .dat decoded without uncorrectable columns stays
        const std::string& path;
        bool armed = true;
        ~Undo() {
            if (armed) unlink(path.c_str());
        }
    } undo{path};
    const int dat_d = fds.keep(open_direct(path, O_WRONLY, direct & 2));
    if (ftruncate(dat, off_t(dat_size)) != 0) return io_fail("size .dat");
    Checked chk{radius, report, ranges, ranges_cap, n_ranges};
    if ((rc = decode_dat(enc.get(), in, in_d, present, dat, dat_d, g, dat_size, g.tail_shard_offset() + g.tail_bytes(0), &chk)))
        return rc;
    if (chk.checked && report->uncorrectable_columns)
        return fail(SWEC_ERR_UNCORRECTABLE, std::to_string(report->uncorrectable_columns) + " byte columns of " + std::string(base) +
                                                " cannot be corrected, shard offsets " + std::to_string(report->first_uncorrectable) +
                                                ".." + std::to_string(report->last_uncorrectable) + ": no .dat written");
    undo.armed = false;
    *ok = chk.checked ? 1 : 0;
    return SWEC_OK;
}

}  // extern "C"
