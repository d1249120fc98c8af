// seaweedfs_b200/csrc/needles.h — the needle record check on the GPU (needles.cu), for host code that stages its own
// records (the volume scrub, ec_volume.cc).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "../../include/swec.h"

namespace swec {

// device scratch a check of n records needs beside its swec_needle_check array (8-byte aligned)
size_t needle_check_scratch_bytes(int n);
// Check n records of the image `dat` (device memory) in place: `checks` is a device array with the inputs filled in;
// asynchronous on `s`, on the current device.
cudaError_t launch_needle_check(const void* dat, int64_t dat_size, int version, swec_needle_check* checks, int n,
                                void* scratch, cudaStream_t s);

}  // namespace swec
