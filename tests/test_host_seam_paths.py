"""Every data path of the Encoder seam (swec_encode, swec_reconstruct, swec_verify and swec_reconstruct_batch on
buffers a cgo reedsolomon.Encoder hands over), across the buffer layouts that pick the path: pageable memory bounced
through the pinned ring, pinned memory DMA'd in place (one strided DMA for slices of one allocation, one DMA per shard
otherwise), calls that mix the two, and shards already in HBM.  Each runs with zero-copy off, on and auto, cut into 1
or 4 pieces, over lengths from 1 B to past one staging chunk, and must give the oracle's bytes without touching the
guard bytes either side of any shard.

The launch fingerprints pin which path each call shape takes: the kernel launches a call makes tell a whole-call
zero-copy launch from a piece-by-piece ring, and a packed batch from the streaming path.  Only matrices compiled into
the library are used (the RS(10,4) parity rows, any single-shard loss, shards 0-3 lost), so the counts never depend
on when a background kernel compile finishes."""
import ctypes as C
import functools

import numpy as np
import pytest

from oracle import rs_numpy

pytestmark = pytest.mark.gpu

K, M, T = 10, 4, 14
GUARD, G = 0x5A, 16  # guard byte value, and guard bytes at least either side of every shard
STAGE_CHUNK = 1 << 20  # small staging chunk for these tests, so that a few MiB span several chunks
# (length, misalignment of every shard)
LENGTHS = ((1, 0), (15, 3), (4096 + 5, 0), (65536, 16), (256 * 1024, 0), ((1 << 20) + 4112, 3), (5 * (1 << 19) + 77, 0))
FP_LENGTHS = ((4096, 0), (256 * 1024 + 5, 0), (65536, 1), (3 * (1 << 20) + 16, 0))
LAYOUTS = ("pageable", "pinned_one_allocation", "pinned_separate", "pinned_in_pageable_out", "pageable_in_pinned_out",
           "half_pinned", "hbm")
DEFAULTS = {"host_zero_copy": 2, "host_pieces": 4, "host_min_chunk": 256 << 10, "stage_chunk": 16 << 20}


def _span(n, shift):
    return (n + shift + 2 * G + 255) & ~255


MAX_SPAN = max(_span(n, s) for n, s in LENGTHS + FP_LENGTHS)


@functools.lru_cache(maxsize=None)
def _shards(n):
    rng = np.random.default_rng(n)
    data = [rng.integers(0, 256, n, dtype=np.uint8) for _ in range(K)]
    return data + rs_numpy.encode(K, M, data)


def _pinned_array(ptr, size):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(size,))


@pytest.fixture(scope="module")
def pinned(cuda, swec):
    """Pinned host memory for the tests: 14 separate allocations, and one allocation for 14 slices."""
    L = swec.lib()
    raws = [L.swec_alloc_pinned_for_device(0, MAX_SPAN) for _ in range(T)] + [L.swec_alloc_pinned_for_device(0, T * MAX_SPAN)]
    try:
        assert all(raws)
        yield [_pinned_array(r, MAX_SPAN) for r in raws[:T]], _pinned_array(raws[T], T * MAX_SPAN)
    finally:
        for r in raws:
            if r:
                L.swec_free_pinned(r)


@pytest.fixture
def options(swec):
    L = swec.lib()

    def set_(name, value):
        assert L.swec_set_option(name.encode(), value) == 0

    try:
        yield set_
    finally:
        for name, value in DEFAULTS.items():
            set_(name, value)


class Shards:
    """The 14 shards of one call, each `n` bytes at `at` inside its own backing buffer of guard bytes."""

    def __init__(self, torch, layout, n, shift, pinned):
        self.n, self.at, self.torch = n, G + shift, torch
        span = _span(n, shift)
        separate, one = pinned
        if layout == "hbm":
            self.backs = [torch.full((span,), GUARD, dtype=torch.uint8, device="cuda") for _ in range(T)]
        elif layout == "pinned_one_allocation":
            self.backs = [one[i * span:(i + 1) * span] for i in range(T)]
        else:
            pin = {"pageable": (), "pinned_separate": range(T), "pinned_in_pageable_out": range(K),
                   "pageable_in_pinned_out": range(K, T), "half_pinned": range(0, T, 2)}[layout]
            # the separate allocations in an order that is not equally spaced, so each shard takes a DMA of its own
            self.backs = [separate[3 * i % T][:span] if i in pin else np.empty(span, dtype=np.uint8) for i in range(T)]
        for b in self.backs:
            if self.device:
                b.fill_(GUARD)
            else:
                b.fill(GUARD)
        self.ptrs = (C.c_void_p * T)(*[self.ptr(i) for i in range(T)])

    @property
    def device(self):
        return not isinstance(self.backs[0], np.ndarray)

    def ptr(self, i):
        b = self.backs[i]
        return (b.data_ptr() if self.device else b.ctypes.data) + self.at

    def get(self, i):
        v = self.backs[i][self.at:self.at + self.n]
        return v.cpu().numpy() if self.device else v.copy()

    def put(self, i, x):
        v = self.backs[i][self.at:self.at + self.n]
        if self.device:
            v.copy_(self.torch.from_numpy(np.ascontiguousarray(x)))
            self.torch.cuda.synchronize()
        else:
            v[:] = x

    def guards_ok(self):
        for b in self.backs:
            whole = b.cpu().numpy() if self.device else b
            if not ((whole[:self.at] == GUARD).all() and (whole[self.at + self.n:] == GUARD).all()):
                return False
        return True


def _launches(L, fn, *args):
    before = L.swec_kernel_launches()
    rc = fn(*args)
    assert rc == 0, L.swec_last_error()
    return int(L.swec_kernel_launches() - before)


def run_layout(L, e, torch, layout, n, shift, pinned):
    """encode, verify (true, then false), reconstruct (shards 0-3 lost, then parity shard 11 lost) and reconstruct_data
    (shards 5 and 12 lost) on one layout, each checked against the oracle; returns the launches of each call."""
    want = _shards(n)
    s = Shards(torch, layout, n, shift, pinned)
    where = (layout, n, shift)
    launches = []
    for i in range(K):
        s.put(i, want[i])
    for i in range(K, T):
        s.put(i, np.full(n, 0xAA, dtype=np.uint8))
    launches.append(_launches(L, L.swec_encode, e._h, s.ptrs, n))
    for i in range(T):
        assert (s.get(i) == want[i]).all(), where + ("encode", i)
    ok = C.c_int(-1)
    launches.append(_launches(L, L.swec_verify, e._h, s.ptrs, n, C.byref(ok)))
    assert ok.value == 1, where
    d0, p3 = want[0].copy(), want[T - 1].copy()
    d0[0] ^= 0xFF
    p3[n - 1] ^= 0xFF
    s.put(0, d0)
    s.put(T - 1, p3)
    launches.append(_launches(L, L.swec_verify, e._h, s.ptrs, n, C.byref(ok)))
    assert ok.value == 0, where
    s.put(0, want[0])
    s.put(T - 1, want[T - 1])
    for lost, data_only in (((0, 1, 2, 3), 0), ((11,), 0), ((5, 12), 1)):
        for i in lost:
            s.put(i, np.zeros(n, dtype=np.uint8))
        present = np.array([i not in lost for i in range(T)], dtype=np.uint8)
        launches.append(_launches(L, L.swec_reconstruct, e._h, s.ptrs, present.ctypes.data, n, data_only))
        for i in lost:
            rebuilt = not data_only or i < K
            assert (s.get(i) == (want[i] if rebuilt else 0)).all(), where + ("reconstruct", lost, i)
            s.put(i, want[i])
    assert s.guards_ok(), where + ("stray write",)
    return launches


@pytest.mark.parametrize("pieces", [1, 4])
@pytest.mark.parametrize("zero_copy", [0, 1, 2])
def test_every_layout_is_bit_exact(cuda, swec, pinned, options, zero_copy, pieces):
    L = swec.lib()
    options("host_zero_copy", zero_copy)
    options("host_pieces", pieces)
    options("host_min_chunk", 4096)
    options("stage_chunk", STAGE_CHUNK)
    e = swec.erasure_coding.Encoder(K, M, device=0)
    try:
        for n, shift in LENGTHS:
            for layout in LAYOUTS:
                run_layout(L, e, cuda, layout, n, shift, pinned)
    finally:
        e.close()


BATCH_LENGTHS = (1, 15, 100, 4096, 65536 + 3, 256 * 1024, (1 << 20) + 5, 2 << 20)


def run_batches(swec, intervals):
    """One reconstruct_batch call over pageable intervals of the given lengths, alternating between a single lost data
    shard and the worst case (shards 0-3 lost), checked against the oracle; returns the call's launches."""
    L = swec.lib()
    e = swec.erasure_coding.Encoder(K, M, device=0)
    try:
        batch, lost_of = [], []
        for j, n in enumerate(intervals):
            want = _shards(n)
            lost = (3,) if j % 2 == 0 else (0, 1, 2, 3)
            batch.append([None if i in lost else want[i].copy() for i in range(T)])
            lost_of.append(lost)
        before = L.swec_kernel_launches()
        e.reconstruct_batch(batch)
        launches = int(L.swec_kernel_launches() - before)
        for shards, lost, n in zip(batch, lost_of, intervals):
            for i in lost:
                assert (shards[i] == _shards(n)[i]).all(), (n, lost, i)
        return launches
    finally:
        e.close()


@pytest.mark.parametrize("zero_copy", [0, 1, 2])
def test_reconstruct_batch_is_bit_exact(cuda, swec, options, zero_copy):
    options("host_zero_copy", zero_copy)
    run_batches(swec, BATCH_LENGTHS)
    run_batches(swec, [4096] * 700)                        # fills slot after slot
    run_batches(swec, [17, (2 << 20) + 1, 4096, 2 << 20])  # one interval over the packed limit streams on its own


def observe_fingerprints(swec, torch, pinned, options):
    """Launches per call for every option setting, layout and fingerprint length, and per batch."""
    L = swec.lib()
    out = {}
    options("host_min_chunk", 4096)
    options("stage_chunk", STAGE_CHUNK)
    for zero_copy in (0, 1, 2):
        options("host_zero_copy", zero_copy)
        for pieces in (1, 4):
            options("host_pieces", pieces)
            e = swec.erasure_coding.Encoder(K, M, device=0)
            try:
                for layout in LAYOUTS:
                    out[f"zc{zero_copy} p{pieces} {layout}"] = " | ".join(
                        " ".join(map(str, run_layout(L, e, torch, layout, n, shift, pinned))) for n, shift in FP_LENGTHS)
            finally:
                e.close()
    options("host_pieces", DEFAULTS["host_pieces"])
    options("host_min_chunk", DEFAULTS["host_min_chunk"])
    options("stage_chunk", DEFAULTS["stage_chunk"])
    for zero_copy in (0, 1, 2):
        options("host_zero_copy", zero_copy)
        out[f"zc{zero_copy} batch"] = " ".join(str(run_batches(swec, lengths)) for lengths in (
            [4096], [100, 65536 + 3], BATCH_LENGTHS, [4096] * 700, [17, (2 << 20) + 1]))
    return out


# launches of encode, verify, verify (mismatch), reconstruct (0-3), reconstruct (11), reconstruct_data (5, 12) at each
# of FP_LENGTHS; for batches, the launches of one reconstruct_batch call per interval list of observe_fingerprints
FINGERPRINTS = {
    "zc0 p1 pageable": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc0 p1 pinned_one_allocation": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc0 p1 pinned_separate": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc0 p1 pinned_in_pageable_out": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc0 p1 pageable_in_pinned_out": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc0 p1 half_pinned": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc0 p1 hbm": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 1 20 20 1 1 1",
    "zc0 p4 pageable": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc0 p4 pinned_one_allocation": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc0 p4 pinned_separate": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc0 p4 pinned_in_pageable_out": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc0 p4 pageable_in_pinned_out": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc0 p4 half_pinned": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc0 p4 hbm": "1 5 5 1 1 1 | 2 21 21 2 2 2 | 1 20 20 1 1 1 | 1 20 20 1 1 1",
    "zc1 p1 pageable": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc1 p1 pinned_one_allocation": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 1 20 20 1 1 1",
    "zc1 p1 pinned_separate": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 1 20 20 1 1 1",
    "zc1 p1 pinned_in_pageable_out": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc1 p1 pageable_in_pinned_out": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc1 p1 half_pinned": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc1 p1 hbm": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 1 20 20 1 1 1",
    "zc1 p4 pageable": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc1 p4 pinned_one_allocation": "1 5 5 1 1 1 | 2 21 21 2 2 2 | 4 20 20 4 4 4 | 1 20 20 1 1 1",
    "zc1 p4 pinned_separate": "1 5 5 1 1 1 | 2 21 21 2 2 2 | 4 20 20 4 4 4 | 1 20 20 1 1 1",
    "zc1 p4 pinned_in_pageable_out": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc1 p4 pageable_in_pinned_out": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc1 p4 half_pinned": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc1 p4 hbm": "1 5 5 1 1 1 | 2 21 21 2 2 2 | 1 20 20 1 1 1 | 1 20 20 1 1 1",
    "zc2 p1 pageable": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc2 p1 pinned_one_allocation": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc2 p1 pinned_separate": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc2 p1 pinned_in_pageable_out": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc2 p1 pageable_in_pinned_out": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc2 p1 half_pinned": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 4 20 20 4 4 4",
    "zc2 p1 hbm": "1 5 5 1 1 1 | 2 6 6 2 2 2 | 1 5 5 1 1 1 | 1 20 20 1 1 1",
    "zc2 p4 pageable": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc2 p4 pinned_one_allocation": "1 5 5 1 1 1 | 2 21 21 2 2 2 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc2 p4 pinned_separate": "1 5 5 1 1 1 | 2 21 21 2 2 2 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc2 p4 pinned_in_pageable_out": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc2 p4 pageable_in_pinned_out": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc2 p4 half_pinned": "1 5 5 1 1 1 | 5 21 21 5 5 5 | 4 20 20 4 4 4 | 4 20 20 4 4 4",
    "zc2 p4 hbm": "1 5 5 1 1 1 | 2 21 21 2 2 2 | 1 20 20 1 1 1 | 1 20 20 1 1 1",
    "zc0 batch": "1 2 3 2 6",
    "zc1 batch": "1 2 3 2 6",
    "zc2 batch": "1 2 3 2 6",
}


def test_launch_fingerprints(cuda, swec, pinned, options):
    got = observe_fingerprints(swec, cuda, pinned, options)
    diff = {k: (v, FINGERPRINTS.get(k)) for k, v in got.items() if v != FINGERPRINTS.get(k)}
    assert not diff, diff
