// seaweedfs_b200/csrc/sketch.h — page sketches of shards (sketch.cu), for the device call and the file call
// (ec_files.cc).  The definition is the one include/swec.h states under SWEC_PAGE_SKETCH_VERSION.
#pragma once
#include <cuda_runtime.h>

#include "apply_params.h"

namespace swec {

// sketches[0 .. ceil(n/4096)) of the n bytes at `shard`, whose first byte is shard offset first_column (a multiple of
// 4096); sketches 8-byte aligned, shard any alignment.  Asynchronous on s; nothing is launched for n = 0.
cudaError_t launch_page_sketch(const void* shard, u64 n, u64 first_column, u64 seed, u64* sketches, cudaStream_t s);

}  // namespace swec
