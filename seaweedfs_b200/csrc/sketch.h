// seaweedfs_b200/csrc/sketch.h — page sketches of shards (sketch.cu), for the device call and the file calls
// (ec_files.cc), and the needles that sketch-located pages hit, for the records-level call and the mounted volume's
// call (ec_volume.cc).  The definition is the one include/swec.h states under SWEC_PAGE_SKETCH_VERSION.
#pragma once
#include <cuda_runtime.h>

#include <vector>

#include "../../include/swec.h"
#include "apply_params.h"
#include "stripe_map.h"

namespace swec {

// sketches[0 .. ceil(n/4096)) of the n bytes at `shard`, whose first byte is shard offset first_column (a multiple of
// 4096); sketches 8-byte aligned, shard any alignment.  Asynchronous on s; nothing is launched for n = 0.
cudaError_t launch_page_sketch(const void* shard, u64 n, u64 first_column, u64 seed, u64* sketches, cudaStream_t s);

// The sketches of the shard files fds (each `size` > 0 bytes, only read) in one pass of the file pipeline on enc's
// device: out[j] (may be NULL) receives the first min(cap, ceil(size/4096)) words of file j.
int page_sketch_files(swec_encoder* enc, const std::vector<int>& fds, int64_t size, uint64_t seed,
                      uint64_t* const* out, int64_t cap);

// The page rules of both sketch needle damage calls (include/swec.h), after pages is known non-NULL when n_pages > 0:
// pages strictly ascending and below ceil(shard_len/4096), uncorrectable 0 or 1, an uncorrectable page with mask 0,
// a blamed page with a non-zero mask below 2^(k+m).  SWEC_ERR_INVALID_ARG naming the first page that breaks one.
int check_sketch_pages(int k, int m, int64_t shard_len, const swec_sketch_page* pages, int64_t n_pages);

// The attribution of both calls, after every check, for n_pages > 0 on `device`: recs[n] (any order; offset and size
// read) get shard_mask, damaged_bytes and uncorrectable_bytes, and unowned the bytes no record owns, for the data
// bytes of the flagged pages mapped by `map`.  Synchronous.
int sketch_needle_damage(int device, const StripeMap& map, int64_t shard_len, const swec_sketch_page* pages,
                         int64_t n_pages, swec_needle_damage* recs, int n, int version, uint64_t unowned[2]);

}  // namespace swec
