// seaweedfs_b200/csrc/host_seam.cc — the Encoder seam on host buffers.
//
// Chunks of every stream travel pinned-host → HBM → kernel → pinned-host on one of a few slots of the encoder's staging
// ring, each with its own stream, so H2D of chunk c+1, the kernel of chunk c and D2H of chunk c-1 overlap.  Caller
// buffers that are already pinned (swec_alloc_pinned / cudaHostRegister) are DMA'd directly; pageable ones bounce
// through the slot's pinned buffer.  Short calls skip the DMA altogether: the kernel reads and writes mapped host
// memory over PCIe itself (zero-copy).
#include "host_seam.h"
#include "io_pool.h"

#include <algorithm>
#include <cstring>
#include <functional>
#include <thread>

namespace swec {

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
static const long g_opt_host_copy_spin_us = long(env_size("SWEC_HOST_COPY_SPIN_US", 200));
static const long g_opt_host_copy_threads = long(env_size("SWEC_HOST_COPY_THREADS", 0));  // 0 = auto

namespace {

// Does this call take zero-copy, for streams of `bytes` each (`cap`: a tighter bound than host_zero_copy_max)?
bool zero_copy_for(size_t bytes, size_t cap = SIZE_MAX) {
    const long mode = g_opt_host_zero_copy.load();
    return mode == 1 || (mode == 2 && bytes <= std::min(size_t(g_opt_host_zero_copy_max.load()), cap));
}

// ---- bounce copies between pageable caller memory and the pinned ring run across a few threads: one core moves
// ~10 GB/s, far less than a PCIe x16 link, so a single memcpy loop would be the whole cost of an Encoder-level call
// from Go heap memory.
struct CopyJob {
    uint8_t* dst;
    const uint8_t* src;
    size_t len;
};

IoPool* host_pool() {  // leaked on purpose (threads must outlive static destructors); nullptr = copy inline
    static IoPool* pool = [] () -> IoPool* {
        long n = g_opt_host_copy_threads;
        if (n <= 0) n = std::min<long>(8, std::max<long>(2, long(std::thread::hardware_concurrency()) / 8));
        return n > 1 ? new IoPool(size_t(n - 1), unsigned(g_opt_host_copy_spin_us)) : nullptr;  // the caller takes a share too
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

// One host call: the encoder's lock and device for all of it.  run() sizes the ring to `chunk` bytes per stream and
// lets pass(turns, &next) queue the pieces, `next` being the slot the next piece takes.  Every slot's turn then
// finishes in submission order from `next` (copy-backs of early pieces overlap the GPU work of late ones); on every
// exit path the slots are drained.
struct SeamCall {
    swec_encoder_impl* e;
    std::lock_guard<std::mutex> lock;
    const int rc;  // of ensure_device: nothing may run unless it is SWEC_OK
    explicit SeamCall(swec_encoder_impl* enc) : e(enc), lock(enc->mu), rc(enc->ensure_device()) {}

    template <class Pass>
    int run(size_t chunk, Pass&& pass) {
        if (const int rc2 = e->ensure_slots(chunk)) return rc2;
        StagingRing& ring = e->ring;
        StagingRing::DrainOnExit drain{ring};
        SlotTurns turns(ring);
        size_t next = 0;
        if (const int rc2 = pass(turns, &next)) return rc2;
        for (size_t i = 0; i < ring.slots.size(); i++)
            if (const int rc2 = turns.finish((next + i) % ring.slots.size())) return rc2;
        return SWEC_OK;
    }
};

// One piece on a slot: the K input streams sit in slot.host at `pitch`, `fill` bytes each.  Either the kernel works on
// the mapped ring itself (reads and writes cross PCIe inside the kernel: one launch instead of H2D + launch + D2H), or
// one strided DMA takes the inputs to slot.dev and one brings the R results back to slot.host at the same pitch.  The
// caller queues the copy-backs out of slot.host.
int run_staged(swec_encoder_impl* e, const Matrix& rows, StagingSlot& s, size_t pitch, size_t fill, bool zero_copy) {
    const int K = rows.cols, R = rows.rows;
    uint8_t* const base = zero_copy ? s.host_dev : s.dev;
    const uint8_t* din[SWEC_MAX_INPUTS];
    uint8_t* dout[SWEC_MAX_SHARDS];
    for (int i = 0; i < K; i++) din[i] = base + size_t(i) * pitch;
    for (int r = 0; r < R; r++) dout[r] = base + size_t(K + r) * pitch;
    if (!zero_copy) SWEC_CUDA(cudaMemcpy2DAsync(s.dev, pitch, s.host, pitch, fill, size_t(K), cudaMemcpyHostToDevice, s.stream));
    if (const int rc = e->apply(rows, din, dout, fill, Layout{}, s.stream)) return rc;
    if (!zero_copy) SWEC_CUDA(cudaMemcpy2DAsync(s.host + size_t(K) * pitch, pitch, dout[0], pitch, fill, size_t(R), cudaMemcpyDeviceToHost, s.stream));
    SWEC_CUDA(cudaEventRecord(s.done, s.stream));
    s.busy = true;
    return SWEC_OK;
}

// What the GPU can reach of one call's K inputs and R outputs (stream s: input s for s < K, output s - K after).
struct CallBuffers {
    bool direct[SWEC_MAX_INPUTS + SWEC_MAX_SHARDS];  // pinned or device memory: DMA'd in place, no bounce
    // the address a kernel uses for the buffer (device memory: itself; mapped pinned host memory: its device alias, the
    // same value under unified addressing), nullptr if a kernel cannot reach it
    uint8_t* gpu[SWEC_MAX_INPUTS + SWEC_MAX_SHARDS];
    bool all_device = true, all_reachable = true, all_pageable = true, all_in_direct = true, all_out_direct = true;

    CallBuffers(const uint8_t* const* in, int K, uint8_t* const* out, int R) {
        uintptr_t align = 0;
        for (int s = 0; s < K + R; s++) {
            cudaPointerAttributes a;
            const bool known = cudaPointerGetAttributes(&a, s < K ? in[s] : out[s - K]) == cudaSuccess;
            if (!known) cudaGetLastError();
            const bool device = known && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged);
            direct[s] = device || (known && a.type == cudaMemoryTypeHost);
            gpu[s] = direct[s] ? static_cast<uint8_t*>(a.devicePointer) : nullptr;
            all_device &= device;
            all_reachable &= gpu[s] != nullptr;
            all_pageable &= !direct[s];
            (s < K ? all_in_direct : all_out_direct) &= direct[s];
            align |= reinterpret_cast<uintptr_t>(gpu[s]);
        }
        all_reachable = all_reachable && (align & 15) == 0;  // the vector kernels need 16-byte aligned streams
    }
};

// p[0..n) equally spaced (the k+m slices of ONE allocation, e.g. swec_alloc_pinned_for_device carved up by the caller)?
bool constant_pitch(const uint8_t* const* p, int n, size_t min_pitch, size_t* pitch) {
    if (n < 2 || p[1] <= p[0]) return false;
    const size_t d = size_t(p[1] - p[0]);
    // cudaMemcpy2D pitches are limited (cudaDevAttrMaxPitch): huge shards go one by one
    if (d < min_pitch || d > size_t(0x7fffffff)) return false;
    for (int i = 2; i < n; i++)
        if (p[i] != p[0] + size_t(i) * d) return false;
    *pitch = d;
    return true;
}

// `rows` rows of `len` bytes, `spitch` apart at src, to `dpitch` apart at dst: one strided DMA.  Equally spaced caller
// buffers are usually slices of one allocation (constant_pitch), but separate pinned allocations can land equally spaced
// too, and the runtime refuses a strided copy whose span is not one pinned range with cudaErrorInvalidValue, before
// anything is queued: then each row goes as a copy of its own.
cudaError_t copy_rows(uint8_t* dst, size_t dpitch, const uint8_t* src, size_t spitch, size_t len, size_t rows,
                      cudaStream_t s) {
    cudaError_t e = cudaMemcpy2DAsync(dst, dpitch, src, spitch, len, rows, cudaMemcpyDefault, s);
    if (e != cudaErrorInvalidValue) return e;
    cudaGetLastError();
    e = cudaSuccess;
    for (size_t r = 0; r < rows && e == cudaSuccess; r++) e = cudaMemcpyAsync(dst + r * dpitch, src + r * spitch, len, cudaMemcpyDefault, s);
    return e;
}

}  // namespace

int apply_host(swec_encoder_impl* e, const Matrix& rows, const uint8_t* const* in, uint8_t* const* out, size_t n,
               unsigned long long* check) {
    const int K = rows.cols, R = rows.rows;
    if (R == 0 || n == 0) return SWEC_OK;
    SeamCall call(e);
    if (call.rc) return call.rc;

    const CallBuffers b(in, K, out, R);
    const bool zero_copy = !check && zero_copy_for(n);
    if (!check && (b.all_device || (zero_copy && b.all_reachable))) {
        // everything already lives in HBM, or every buffer is mapped pinned (or device) memory: ONE launch reads the
        // data shards (over PCIe) and writes the parity back; what a 256 KiB-per-shard Encode call costs is this
        // launch and one stream synchronise
        const uint8_t* const* kin = b.all_device ? in : b.gpu;
        uint8_t* const* kout = b.all_device ? out : b.gpu + K;
        if (const int rc = e->apply(rows, kin, kout, n, Layout{}, e->stream)) return rc;
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

    // pinned callers whose k+m buffers are slices of one allocation: ONE strided DMA each way instead of k + m
    size_t in_pitch = 0, out_pitch = 0;
    const bool in_2d = b.all_in_direct && constant_pitch(in, K, n, &in_pitch);
    const bool out_2d = !check && b.all_out_direct && R > 1 && constant_pitch(out, R, n, &out_pitch);
    const bool packed = !check && b.all_pageable;

    // verify's count of mismatching vectors, zeroed before any slot stream compares into it; it outlives run(), which
    // drains every slot on its way out
    StreamScratch dev_bad(e->stream);
    const int rc = call.run(chunk, [&](SlotTurns& turns, size_t* next) -> int {
        if (check) {
            SWEC_CUDA(dev_bad.alloc(8));
            SWEC_CUDA(cudaMemsetAsync(dev_bad.p, 0, 8, e->stream));
            SWEC_CUDA(cudaStreamSynchronize(e->stream));
        }
        StagingRing& ring = e->ring;
        const size_t stride = e->slot_chunk();  // per-stream pitch inside a slot (>= chunk)
        std::vector<CopyJob> bounce;
        for (size_t off = 0; off < n; off += chunk) {
            const size_t si = *next;
            StagingSlot& s = ring.slots[si];
            if (const int rc2 = turns.finish(si)) return rc2;
            *next = (si + 1) % ring.slots.size();
            const size_t len = std::min(chunk, n - off);
            // Pageable callers (Go heap memory) bounce through the slot anyway, so pack the streams at a
            // pitch that fits this piece: one DMA in, one DMA out instead of k + m small ones.
            const size_t pitch = packed ? ((len + 255) & ~size_t(255)) : stride;
            bounce.clear();
            for (int i = 0; i < K; i++)
                if (!b.direct[i]) bounce.push_back({s.host + size_t(i) * pitch, in[i] + off, len});
            parallel_copy(bounce);
            if (packed) {
                if (const int rc2 = run_staged(e, rows, s, pitch, len, zero_copy && s.host_dev)) return rc2;
                for (int r = 0; r < R; r++) turns.pending[si].push_back({out[r] + off, s.host + size_t(K + r) * pitch, len});
                continue;
            }
            const uint8_t* din[SWEC_MAX_INPUTS];
            uint8_t* dout[SWEC_MAX_SHARDS];
            for (int i = 0; i < K; i++) din[i] = s.dev + size_t(i) * pitch;
            for (int r = 0; r < R; r++) dout[r] = s.dev + size_t(K + r) * pitch;
            if (in_2d) {
                SWEC_CUDA(copy_rows(s.dev, pitch, in[0] + off, in_pitch, len, size_t(K), s.stream));
            } else {
                for (int i = 0; i < K; i++) {
                    const uint8_t* src = b.direct[i] ? in[i] + off : s.host + size_t(i) * pitch;
                    SWEC_CUDA(cudaMemcpyAsync(s.dev + size_t(i) * pitch, src, len, cudaMemcpyDefault, s.stream));
                }
            }
            if (const int rc2 = e->apply(rows, din, dout, len, Layout{}, s.stream)) return rc2;
            if (out_2d) {
                SWEC_CUDA(copy_rows(out[0] + off, out_pitch, dout[0], pitch, len, size_t(R), s.stream));
            } else {
                if (check) {  // bring the caller's copy of every row next to the computed one and compare in HBM
                    bounce.clear();
                    for (int r = 0; r < R; r++)
                        if (!b.direct[K + r]) bounce.push_back({s.host + size_t(K + r) * stride, out[r] + off, len});
                    parallel_copy(bounce);
                }
                for (int r = 0; r < R; r++) {
                    const bool direct = b.direct[K + r];
                    if (check) {
                        uint8_t* theirs = s.dev + size_t(K + R + r) * stride;
                        const uint8_t* src = direct ? out[r] + off : s.host + size_t(K + r) * stride;
                        SWEC_CUDA(cudaMemcpyAsync(theirs, src, len, cudaMemcpyDefault, s.stream));
                        SWEC_CUDA(launch_compare(dout[r], theirs, len, dev_bad.as<unsigned long long>(), s.stream));
                    } else if (direct) {
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
        return SWEC_OK;
    });
    if (!rc && check && cudaMemcpy(check, dev_bad.p, 8, cudaMemcpyDeviceToHost) != cudaSuccess)
        return cuda_fail(cudaGetLastError(), "reading the mismatch counter");
    return rc;
}

// Largest interval the packed path takes (bigger ones stream through apply_host): small on purpose — the
// ring behind it is 3 slots x (k+2m) streams x this, and needle-sized intervals gain nothing from more.
size_t packed_max_bytes() { return std::min(size_t(std::max(4096l, g_opt_stage_chunk.load())), size_t(2) << 20); }

int apply_host_packed(swec_encoder_impl* e, const Matrix& rows, const std::vector<Segment>& segs) {
    const int K = rows.cols, R = rows.rows;
    if (R == 0 || segs.empty()) return SWEC_OK;
    SeamCall call(e);
    if (call.rc) return call.rc;
    // size the ring for THIS batch (a lone degraded read must not pin 3 x 18 x 16 MiB): everything packed
    // back to back, capped by the configured chunk; ensure_slots only ever grows an existing ring
    size_t packed = 0;
    for (const Segment& sg : segs) packed += (sg.len + 15) & ~size_t(15);
    const size_t chunk = std::min(packed_max_bytes(), (packed + 65535) & ~size_t(65535));
    return call.run(chunk, [&](SlotTurns& turns, size_t* si) -> int {
        StagingRing& ring = e->ring;
        const size_t stride = e->slot_chunk();
        size_t fill = 0;
        auto flush = [&]() -> int {
            if (fill == 0) return SWEC_OK;
            StagingSlot& sl = ring.slots[*si];
            // the K input streams sit at pitch `stride` in the slot.  Zero-copy pays for one needle per call and costs
            // when many needles fill slot after slot (earlier GPU generation; scripts/bench_needles.py measures it):
            // full slots keep the strided-DMA pipeline.
            const int rc = run_staged(e, rows, sl, stride, fill, zero_copy_for(fill, size_t(256) << 10) && sl.host_dev);
            if (rc) return rc;
            fill = 0;
            *si = (*si + 1) % ring.slots.size();
            return turns.finish(*si);  // the slot we are about to fill must be drained
        };
        for (const Segment& sg : segs) {
            const size_t padded = (sg.len + 15) & ~size_t(15);
            // larger than a slot: not a "small interval" — the caller should not batch it
            if (padded > stride) return fail(SWEC_ERR_INVALID_ARG, "batched interval larger than the staging chunk");
            if (fill + padded > stride)
                if (const int rc = flush()) return rc;
            StagingSlot& sl = ring.slots[*si];
            for (int i = 0; i < K; i++) {
                uint8_t* dst = sl.host + size_t(i) * stride + fill;
                memcpy(dst, sg.in[i], sg.len);
                if (padded > sg.len) memset(dst + sg.len, 0, padded - sg.len);
            }
            for (int r = 0; r < R; r++) turns.pending[*si].push_back({sg.out[r], sl.host + size_t(K + r) * stride + fill, sg.len});
            fill += padded;
        }
        return flush();
    });
}

}  // namespace swec
