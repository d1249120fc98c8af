// seaweedfs_b200/csrc/host_seam.h — the Encoder seam on host buffers: what swec_encode, swec_reconstruct, swec_verify
// and swec_reconstruct_batch run when a cgo reedsolomon.Encoder hands over Go heap or pinned memory.
#pragma once
#include "engine.h"

namespace swec {

// "host_pieces", "host_min_chunk", "host_zero_copy", "host_zero_copy_max": see host_seam.cc
extern std::atomic<long> g_opt_host_pieces, g_opt_host_min_chunk, g_opt_host_zero_copy, g_opt_host_zero_copy_max;

// out[r] = rows ⊗ in over n bytes of host (or device) buffers, synchronous.  check != nullptr: out[r] are read and
// compared with the computed rows instead; *check receives the number of mismatching 16-byte vectors.
int apply_host(swec_encoder_impl* e, const Matrix& rows, const uint8_t* const* in, uint8_t* const* out, size_t n,
               unsigned long long* check);

// Many small intervals that share one matrix (degraded reads behind one dead server), packed back to back (each padded
// to 16 bytes) into slot-sized launches: the per-call costs — stream round trip, launch, DMA set-up — are paid once
// per ~chunk instead of once per needle.  packed_max_bytes(): the largest padded interval it takes.
struct Segment {
    std::vector<const uint8_t*> in;  // K pointers
    std::vector<uint8_t*> out;       // R pointers
    size_t len;
};
int apply_host_packed(swec_encoder_impl* e, const Matrix& rows, const std::vector<Segment>& segs);
size_t packed_max_bytes();

}  // namespace swec
