// seaweedfs_b200/csrc/staging.h — pinned host memory near the GPU, and the staging ring host data travels through on
// its way to the kernels and back: the Encoder seam (host_seam.cc) and the file pipelines (ec_files.cc) each use one.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

namespace swec {

// the NUMA node the GPU hangs off; -1 when unknown, beyond what an mbind mask here holds, or SWEC_NO_NUMA is set
int device_numa_node(int device);
// MPOL_PREFERRED: [p, p+len) stays on `node` while it has room, never failing the allocation (node < 0: no-op)
void bind_to_node(void* p, size_t len, int node);
// cudaHostRegister (portable, mapped) of an mmap'ed range, which pinned_free then unregisters and unmaps
cudaError_t register_mapped(void* p, size_t len);
// pinned, mapped host memory on the NUMA node of `device` (plain cudaHostAlloc when that is unknown)
void* pinned_alloc(int device, size_t bytes);
void pinned_free(void* p);

struct StagingSlot {
    uint8_t* host = nullptr;      // pinned
    uint8_t* host_dev = nullptr;  // the same memory as the GPU addresses it (mapped pinned memory), or nullptr
    uint8_t* dev = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    bool busy = false;  // work queued on `stream` may still touch the slot or the caller's buffers
};

struct StagingRing {
    int device = -1;
    size_t bytes_per_slot = 0;
    std::vector<StagingSlot> slots;  // empty: no ring

    // n slots of `bytes` pinned and `bytes` device memory each, replacing any ring held before.  All or nothing: a
    // half-built ring must never look big enough.
    int allocate(int device, size_t n, size_t bytes);
    void release();  // synchronise every slot's stream and free everything
    void drain();    // wait for every busy slot and mark it free

    // Whatever way a host-path call ends, no DMA may still be aimed at the caller's buffers when it returns
    // ("nothing is retained after a call returns", include/swec.h).
    struct DrainOnExit {
        StagingRing& ring;
        ~DrainOnExit() { ring.drain(); }
    };
};

}  // namespace swec
