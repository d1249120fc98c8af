"""The Encoder seam on shards that are equally spaced in memory but pinned as separate registrations.

The seam moves the k+m streams of a pinned caller with one strided DMA when they are equally spaced, which is what the
slices of one allocation look like.  Separate pinned allocations can land equally spaced too (the placement of a run of
pinned allocations depends on what the process mapped and unmapped before), and the runtime refuses a strided copy whose
span is not one pinned range.  Here the caller's buffers are carved out of one pageable array and each shard is
registered on its own, with and without unregistered gaps between them, so the strided path meets that case on purpose:
encode and reconstruct must give the oracle's bytes without touching the gaps."""
import ctypes as C

import numpy as np
import pytest

from oracle import rs_numpy
from test_host_seam_paths import DEFAULTS

pytestmark = pytest.mark.gpu

K, M, T = 10, 4, 14
SLOT = 1 << 20          # bytes between the starts of two registered shards' slots
GUARD = 0x5A


@pytest.fixture
def dma_only(swec):
    """Zero-copy off, so every call takes the DMA ring and its strided copies; the defaults come back afterwards."""
    L = swec.lib()
    for name, value in (("host_zero_copy", 0), ("host_min_chunk", 4096)):
        assert L.swec_set_option(name.encode(), value) == 0
    try:
        yield L
    finally:
        for name, value in DEFAULTS.items():
            assert L.swec_set_option(name.encode(), value) == 0


class Region:
    """One page-aligned pageable array; shard i at offset i * stride, registered (pinned) one shard at a time."""

    def __init__(self, torch, stride, registered):
        self.cudart = torch.cuda.cudart()
        self.raw = np.full(T * stride + 4096, GUARD, dtype=np.uint8)
        self.base = (-self.raw.ctypes.data) % 4096
        self.stride, self.done = stride, []
        for i in registered:
            rc = self.cudart.cudaHostRegister(self.ptr(i), SLOT, 3)     # portable | mapped
            assert rc == self.cudart.cudaError.success, (i, rc)
            self.done.append(i)

    def ptr(self, i):
        return self.raw.ctypes.data + self.base + i * self.stride

    def view(self, i, n):
        return self.raw[self.base + i * self.stride:self.base + i * self.stride + n]

    def close(self):
        for i in self.done:
            self.cudart.cudaHostUnregister(self.ptr(i))
        self.done = []


@pytest.mark.parametrize("stride,registered", [(2 * SLOT, range(K, T)), (2 * SLOT, range(T)), (SLOT, range(T))],
                         ids=["parity_pinned_with_gaps", "all_pinned_with_gaps", "all_pinned_adjacent"])
def test_equally_spaced_separate_pins(cuda, swec, dma_only, stride, registered):
    L = dma_only
    n = 300_000 + 7
    rng = np.random.default_rng(stride + len(registered))
    data = [rng.integers(0, 256, n, dtype=np.uint8) for _ in range(K)]
    want = data + rs_numpy.encode(K, M, data)
    enc = swec.erasure_coding.Encoder(K, M, device=0)
    r = Region(cuda, stride, registered)
    try:
        ptrs = (C.c_void_p * T)(*[r.ptr(i) for i in range(T)])
        for i in range(K):
            r.view(i, n)[:] = data[i]
        assert L.swec_encode(enc._h, ptrs, n) == 0, L.swec_last_error()
        for i in range(T):
            assert (r.view(i, n) == want[i]).all(), i
        lost = (0, 1, 2, 3)                 # the rebuilt data shards are equally spaced outputs too
        for i in lost:
            r.view(i, n)[:] = 0
        present = np.array([i not in lost for i in range(T)], dtype=np.uint8)
        assert L.swec_reconstruct(enc._h, ptrs, present.ctypes.data, n, 0) == 0, L.swec_last_error()
        for i in range(T):
            assert (r.view(i, n) == want[i]).all(), i
        for i in range(T):                  # nothing outside the shards was written
            gap = r.raw[r.base + i * stride + n:r.base + (i + 1) * stride]
            assert (gap == GUARD).all(), i
    finally:
        r.close()
        enc.close()
