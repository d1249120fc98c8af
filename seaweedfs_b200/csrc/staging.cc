// seaweedfs_b200/csrc/staging.cc — pinned host memory near the GPU, and the staging ring (staging.h).
#include "staging.h"
#include "engine.h"

#include <cstdio>

#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

namespace swec {

// ------------------------------------------------------------------ NUMA-local pinned host memory
// PCIe DMA from the far socket costs ~15-20 % of H2D bandwidth on two-socket hosts, so staging
// memory is bound (mbind) to the NUMA node the GPU hangs off before it is pinned.

static std::mutex g_pin_mu;
static std::map<void*, size_t> g_pin_mapped;  // regions we mmap'ed + registered

int device_numa_node(int device) {
    if (getenv("SWEC_NO_NUMA")) return -1;
    char bus[32] = {0};
    if (device < 0 || cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    for (char* c = bus; *c; c++) *c = char(tolower(*c));
    const std::string path = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
    FILE* f = fopen(path.c_str(), "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node < 1024 ? node : -1;
}

void bind_to_node(void* p, size_t len, int node) {
    if (node < 0) return;
    unsigned long mask[16] = {0};
    mask[size_t(node) / (8 * sizeof(unsigned long))] |= 1ul << (size_t(node) % (8 * sizeof(unsigned long)));
    syscall(SYS_mbind, p, len, 1 /* MPOL_PREFERRED */, mask, sizeof(mask) * 8, 0);
}

cudaError_t register_mapped(void* p, size_t len) {
    const cudaError_t e = cudaHostRegister(p, len, cudaHostRegisterPortable | cudaHostRegisterMapped);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lk(g_pin_mu);
    g_pin_mapped[p] = len;
    return cudaSuccess;
}

// Pinned staging memory is carved out of 2 MiB-aligned anonymous mappings with MADV_HUGEPAGE: when several GPUs of one
// socket DMA concurrently, every 4 KiB page is its own translation for the root complex / IOMMU, and the pages of a
// huge page are physically contiguous, which DMA engines split less.  Best effort (the kernel may have THP off);
// SWEC_NO_THP=1 keeps plain 4 KiB pages for A/B measurements.
static void* map_aligned(size_t len, size_t* mapped_len) {
    const size_t huge = size_t(2) << 20;
    const bool thp = !getenv("SWEC_NO_THP") && len >= huge;
    const size_t want = thp ? ((len + huge - 1) & ~(huge - 1)) : len;
    const size_t span = thp ? want + huge : want;
    uint8_t* raw = static_cast<uint8_t*>(mmap(nullptr, span, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0));
    if (raw == MAP_FAILED) return nullptr;
    uint8_t* p = raw;
    if (thp) {
        p = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + huge - 1) & ~uintptr_t(huge - 1));
        if (p > raw) munmap(raw, size_t(p - raw));
        const size_t tail = size_t(raw + span - (p + want));
        if (tail) munmap(p + want, tail);
        madvise(p, want, MADV_HUGEPAGE);
    }
    *mapped_len = want;
    return p;
}

void* pinned_alloc(int device, size_t bytes) {
    if (bytes == 0) return nullptr;
    const int node = device_numa_node(device);
    if (node >= 0) {
        size_t len = (bytes + 4095) & ~size_t(4095);
        void* p = map_aligned(len, &len);
        if (p) {
            bind_to_node(p, len, node);
            if (register_mapped(p, len) == cudaSuccess) return p;
            cudaGetLastError();
            munmap(p, len);
        }
    }
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocPortable | cudaHostAllocMapped) != cudaSuccess) {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}

void pinned_free(void* p) {
    if (!p) return;
    size_t len = 0;
    {
        std::lock_guard<std::mutex> lk(g_pin_mu);
        auto it = g_pin_mapped.find(p);
        if (it != g_pin_mapped.end()) {
            len = it->second;
            g_pin_mapped.erase(it);
        }
    }
    if (len) {
        cudaHostUnregister(p);
        munmap(p, len);
    } else {
        cudaFreeHost(p);
    }
}

// ------------------------------------------------------------------ the staging ring

int StagingRing::allocate(int dev, size_t n, size_t bytes) {
    release();
    device = dev;
    bytes_per_slot = bytes;
    slots.resize(n);
    for (StagingSlot& s : slots) {
        s.host = static_cast<uint8_t*>(pinned_alloc(device, bytes));
        cudaError_t e = s.host ? cudaSuccess : cudaErrorMemoryAllocation;
        if (e == cudaSuccess && cudaHostGetDevicePointer(reinterpret_cast<void**>(&s.host_dev), s.host, 0) != cudaSuccess) {
            cudaGetLastError();
            s.host_dev = nullptr;  // not mapped: the slot still works through DMA
        }
        if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&s.dev), bytes);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming);
        if (e != cudaSuccess) {
            const bool no_host = !s.host;
            release();
            cudaGetLastError();
            return no_host ? fail(SWEC_ERR_NOMEM, "cannot allocate pinned staging memory") : cuda_fail(e, "allocating the staging ring");
        }
    }
    return SWEC_OK;
}

void StagingRing::release() {
    if (!slots.empty() && cudaSetDevice(device) != cudaSuccess) cudaGetLastError();
    for (StagingSlot& s : slots) {
        if (s.stream) cudaStreamSynchronize(s.stream);
        if (s.host) pinned_free(s.host);
        if (s.dev) cudaFree(s.dev);
        if (s.done) cudaEventDestroy(s.done);
        if (s.stream) cudaStreamDestroy(s.stream);
    }
    slots.clear();
    bytes_per_slot = 0;
}

void StagingRing::drain() {
    for (StagingSlot& s : slots)
        if (s.busy) {
            if (s.stream) cudaStreamSynchronize(s.stream);
            s.busy = false;
        }
}

}  // namespace swec
