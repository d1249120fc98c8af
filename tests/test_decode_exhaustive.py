"""The checked decode (swec_decode_data_checked_device, and the file-level calls built on it) at every syndrome of the
small codes, at radius 2, and on every code shape the encoder accepts.

ec.decode deletes every shard, parity included, once the .dat is written, so this decode is the last chance to correct
a damaged data shard.  It runs on kDecode, the fourth mode of swec_locate_kernel (damage.cu): the rebuild mode, with rows
only for the missing data shards, plus restore(), which XORs each located error value of an information position that
holds a data shard into that shard's own byte.  The sweeps build their inputs as tests/test_damage_exhaustive.py does
(a syndrome XORed into the stored check rows of a tiled random codeword, the blame looked up in the exhaustive error
table of tests/damage_oracle.py) and compare the whole report and every byte of every buffer with what the decode must
leave (expected_decode): present data corrected by the blamed values, missing data rebuilt (plain rebuild XOR the images
R[row][j]·e_j of the blamed information errors), every parity byte as it was, a missing parity shard's buffer (or NULL)
untouched, and the padding around shifted pointers kept.

cpu: expected_decode equals the independent oracle test_checked_decode.checked_decode, bytes and report, on fuzzed sets
of RS(10,4) (nothing, a data shard, a parity shard, a data + parity pair lost), RS(8,6) (shard 3 or 9 lost), RS(16,16)
(14 data shards lost) and RS(1,3) (shard 0 lost); the swec_locate_kernel instantiations in libswec.so are exactly the
nine of LEDGER.
gpu, syndrome sweeps:
  - RS(10,4) nothing lost (c = 4), radius 1 and 2: all 4,294,967,295 non-zero syndromes, 16 calls of 2^28 columns;
  - RS(10,4) single losses (c = 3) at all 16,777,215 check syndromes, radius 0, 1, 2; double losses (c = 2) at all
    65,535, radius 0 and 1; each report also equals the checked rebuild's on the same shards;
  - RS(10,4) triple losses (c = 1) at all 255 syndromes: uncorrectable, the data of a data-only reconstruct; quadruple
    losses (c = 0): nothing checked, the data of a data-only reconstruct;
  - m = 2 and 3, radius 1, every non-zero syndrome of RS(3,2), RS(30,2), RS(1,3), RS(6,3), RS(29,3), aligned with a
    7-column tail and at pointer offset 3, and RS(1,3) with shard 0 lost (its only information shard is parity);
  - RS(8,6) at radius 2 (any c): nothing lost, all 5,920,845 patterns of 1 or 2 wrong shards and 2^24 random
    syndromes; shard 3 lost and shard 9 lost, all 5,075,265 patterns each;
  - every radius-2 syndrome with each byte cleared in turn: RS(5,5) nothing lost, RS(8,6) shard 3 lost;
  - one RS(10,4) call of 2^28 + 4,103 columns with shard 2 lost: damage on both sides of the 256 MiB piece boundary.
gpu, the include/swec.h guarantee against injected damage (not a table) on RS(1,2) ... RS(16,16) at radius 0, 1 and 2,
with nothing, one data, one parity, m-2 and m-4 mixed shards lost (and 14 data shards of RS(16,16)), aligned and at
offset 3; file level at RS(20,12) radius 2 with (5, 13) and (5, 27) lost; which swec_locate_kernel instantiation each
sweep's configuration runs, and every one of LEDGER, recorded with torch.profiler in a child process."""
import itertools
import json
import os
import re
import shutil
import subprocess
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import damage_oracle as do  # noqa: E402
import test_checked_decode as tcd  # noqa: E402
import test_checked_rebuild as tcr  # noqa: E402
import test_damage_exhaustive as tde  # noqa: E402
import test_kernel_variants as tkv  # noqa: E402

from oracle import rs_numpy as rn  # noqa: E402

FILL = 0xA5        # a missing data shard's buffer before the call: every byte of it must be written
SENTINEL = 0x5A    # a missing parity shard's buffer: never written
LOCATE, CORRECT, REBUILD, DECODE = 0, 1, 2, 3   # the MODE template argument of swec_locate_kernel
# every (MT, MODE) instantiation of swec_locate_kernel; MT = 0 is the run-time m (c for rebuild and decode)
LEDGER = {(4, LOCATE), (0, LOCATE), (4, CORRECT), (0, CORRECT), (3, REBUILD), (0, REBUILD), (4, DECODE), (3, DECODE),
          (0, DECODE)}


def decode_id(c):
    return (c if c in (3, 4) else 0, DECODE)


def rebuild_id(c):
    return (3 if c == 3 else 0, REBUILD)


def locate_id(name):
    """(MT, MODE) of a swec_locate_kernel from its mangled or demangled name, else None."""
    m = re.search(r"swec_locate_kernelILi(\d+)ELi(\d+)E", name) or re.search(r"swec_locate_kernel<(\d+), ?(\d+)>", name)
    return (int(m[1]), int(m[2])) if m else None


# ------------------------------------------------------------------------------------------ expected values


def expected_decode(torch, before, shift, length, k, m, present, a, b, va, vb, damaged, plain):
    """(the buffer, the report) a decode leaves on `before` (n rows, shard i at columns [shift, shift + length)) when
    column x is blamed on positions a, b (-1: none) with values va, vb: a present data shard at information position p
    gets the values blamed on p XORed in, missing data shard i is plain[i] (the plain rebuild from the information set
    as found) XOR the images R[row][j]·e_j of the blamed information errors, every other byte stays as it was."""
    info, checks, lost, _, r = do.punctured_rows(k, m, tuple(present))
    ids = info + checks
    want = tde.without_ok(do.dense_report(tde.to_ids(torch, ids, a), tde.to_ids(torch, ids, b), damaged, k + m))
    out = before.clone()
    for p, sid in enumerate(info):
        if sid < k:
            out[sid, shift:shift + length] ^= torch.where(a == p, va, 0) ^ torch.where(b == p, vb, 0)
    mul = tde.gmul_table(torch)
    for row, i in enumerate(lost):
        if i < k:
            coef = torch.zeros(k + len(checks) + 1, dtype=torch.uint8, device=tde.DEV)   # by position + 1
            coef[1:k + 1] = torch.from_numpy(r[row]).to(tde.DEV)
            out[i, shift:shift + length] = (plain[i] ^ tde.gmul(mul, coef[a.long() + 1], va)
                                            ^ tde.gmul(mul, coef[b.long() + 1], vb))
    return out, want


def fill_lost(buf, k, lost):
    for i in lost:
        buf[i].fill_(FILL if i < k else SENTINEL)


def decode_ptrs(buf, shift, k, lost, null_parity):
    p = tde.ptrs(buf, shift)
    for i in lost:
        if i >= k and null_parity:
            p[i] = None
    return p


def check_decode(torch, enc, buf, shift, length, k, m, present, radius, a, b, va, vb, damaged, plain,
                 null_parity=False, rebuild=False):
    """Decode `buf` (clean but for the injected syndromes; plain: the clean bytes of the missing data shards) and
    compare every byte and the report with expected_decode; `rebuild`: the checked rebuild of a copy reports the same."""
    lost = [i for i in range(k + m) if not present[i]]
    fill_lost(buf, k, lost)
    want_buf, want = expected_decode(torch, buf, shift, length, k, m, present, a, b, va, vb, damaged, plain)
    copy = buf.clone() if rebuild else None
    got = enc.decode_data_checked_device(decode_ptrs(buf, shift, k, lost, null_parity), [int(x) for x in present],
                                         length, radius=radius, max_ranges=tde.MAX_RANGES)
    assert got == want, (present, radius)
    assert torch.equal(buf, want_buf), (present, radius)
    del want_buf
    if rebuild:
        assert enc.reconstruct_checked_device(tde.ptrs(copy, shift), present, length, radius=radius,
                                              max_ranges=tde.MAX_RANGES) == got, (present, radius)
    return got


def inject_keys(torch, buf, rows, shift, keys):
    """XOR byte i of every column's key into rows[i]"""
    length = len(keys)
    for i, r in enumerate(rows):
        buf[r, shift:shift + length] ^= ((keys >> (8 * i)) & 255).to(torch.uint8)


# ------------------------------------------------------------------------------------------ CPU

BUILDER_CASES = [(10, 4, ()), (10, 4, (3,)), (10, 4, (12,)), (10, 4, (2, 11)), (8, 6, (3,)), (8, 6, (9,)),
                 (16, 16, tuple(range(1, 15))), (1, 3, (0,))]


@pytest.mark.parametrize("k,m,lost", BUILDER_CASES)
def test_expected_values_equal_the_checked_decode_oracle(monkeypatch, k, m, lost):
    """expected_decode, given the oracle's blame, writes the data shards and builds the report that
    test_checked_decode.checked_decode computes independently, and leaves parity, fill and padding alone."""
    import torch
    monkeypatch.setattr(tde, "DEV", "cpu")
    n, length, shift = k + m, 3001, 3
    present = tde.mask(n, lost)
    info, checks, _, _, r = do.punctured_rows(k, m, present)
    c = len(checks)
    shards = tde.fuzz(k, m, length, c, seed=n * 10 + len(lost), present=present)
    found = [s if present[i] else None for i, s in enumerate(shards)]
    before = tde.buffer(torch, n, length, shift)
    before[:, :shift] = 7
    for i in range(n):
        before[i, shift:shift + length] = torch.from_numpy(shards[i])
    fill_lost(before, k, lost)
    plain = {i: torch.from_numpy(v) for i, v in zip(lost, rn.apply_rows(r, [shards[j] for j in info])) if i < k}
    for radius in (0, 1, 2):
        cols, pa, pb, pva, pvb, _ = do.decode_columns(shards, k, m, min(radius, c // 2), present)
        a, b = (torch.full((length,), -1, dtype=torch.int8) for _ in range(2))
        va, vb = (torch.zeros(length, dtype=torch.uint8) for _ in range(2))
        for dst, src in ((a, pa), (b, pb), (va, pva), (vb, pvb)):
            dst[torch.from_numpy(cols)] = torch.from_numpy(src).to(dst.dtype)
        damaged = torch.zeros(length, dtype=torch.bool)
        damaged[torch.from_numpy(cols)] = True
        got, rep = expected_decode(torch, before, shift, length, k, m, present, a, b, va, vb, damaged, plain)
        want_data, want = tcd.checked_decode(found, k, m, present, radius)
        assert rep == tde.without_ok(want), radius
        assert rep["damaged_columns"] > 0 and (radius == 0 or len(rep["shards"]) > 0), radius
        for i in range(k):
            assert (got[i, shift:shift + length].numpy() == want_data[i]).all(), (radius, i)
        keep = [i for i in range(n) if i >= k]
        assert torch.equal(got[keep], before[keep]), radius
        assert torch.equal(got[:, :shift], before[:, :shift]) and torch.equal(got[:, shift + length:],
                                                                              before[:, shift + length:])


def test_locate_ledger_matches_the_library(swec):
    """The swec_locate_kernel instantiations in libswec.so are exactly LEDGER, which the GPU part launches by name: a
    new instantiation fails here until a test launches it."""
    from seaweedfs_b200 import _native
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("no CUDA toolkit")
    out = subprocess.run([cuobjdump, "-symbols", _native.library_path()], capture_output=True, text=True,
                         check=True).stdout
    found = {locate_id(ln.split()[-1]) for ln in out.splitlines() if "STT_FUNC" in ln and "STO_ENTRY" in ln}
    found.discard(None)
    assert found == LEDGER, {"not launched": sorted(found - LEDGER), "not in the library": sorted(LEDGER - found)}


def test_locate_id_reads_both_spellings():
    assert locate_id("_ZN4swec41_GLOBAL__N__e409e7bd_9_damage_cu_e5cab04218swec_locate_kernelILi4ELi3EEEvNS0_"
                     "12LocateParamsE") == locate_id("void swec::(anonymous namespace)::swec_locate_kernel<4, 3>("
                                                     "swec::(anonymous namespace)::LocateParams)") == (4, DECODE)
    assert locate_id("void at::native::fill_kernel") is None


# ------------------------------------------------------------------------------------------ GPU: syndrome sweeps


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [1, 2])
def test_decode_every_syndrome_of_rs_10_4(cuda, swec, radius):
    """Nothing lost (c = 4): all 2^32 syndromes, 2^28 columns a call: column x of slice s carries s·2^28 + x."""
    torch = cuda
    if tde.free_bytes(torch) < 16 * tde.GIB:
        pytest.skip("needs 16 GiB of free device memory")
    k, m = 10, 4
    n_slice = 1 << tde.SLICE_BITS
    present = tde.mask(k + m, ())
    table = do.error_table(k, m, radius, present)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    clean = tde.tiled(torch, k, m, n_slice, seed=1043)
    blamed = uncorrectable = 0
    times = []
    for s in range(1 << (32 - tde.SLICE_BITS)):
        t0 = time.perf_counter()
        buf = clean.clone()
        keys = tde.inject_counting(torch, buf, range(k, k + m), 0, n_slice, tde.SLICE_BITS, lo=s << tde.SLICE_BITS)
        a, b, va, vb = tde.blame(torch, table, keys)
        got = check_decode(torch, enc, buf, 0, n_slice, k, m, present, radius, a, b, va, vb, keys != 0, {})
        blamed += int((a >= 0).sum())
        uncorrectable += got["uncorrectable_columns"]
        del buf, keys, a, b, va, vb
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    assert blamed == len(table[0]) and blamed + uncorrectable == (1 << 32) - 1
    print(f"\nRS(10,4) decode radius {radius}: 16 slices of 2^28 columns, "
          f"{min(times):.2f} .. {max(times):.2f} s a slice, {sum(times):.1f} s in all")


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [0, 1, 2])
def test_decode_every_check_syndrome_of_rs_10_4_with_losses(cuda, swec, radius):
    """14 single losses x 2^24 check syndromes (c = 3, radius 2 clamps to 1); at radius 0 and 1 also 91 double losses
    x 2^16 (c = 2).  With a data shard lost, parity 10 is an information position: its blamed errors reach the rebuilt
    shard and never shard 10.  Each report equals the checked rebuild's; a missing parity shard alternates between a
    NULL pointer and a sentinel buffer."""
    torch = cuda
    k, m = 10, 4
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    for f in (1, 2) if radius < 2 else (1,):
        c = m - f
        length = 1 << (8 * c)
        clean = tde.tiled(torch, k, m, length, seed=20 + f)
        for n_case, lost in enumerate(itertools.combinations(range(k + m), f)):
            present = tde.mask(k + m, lost)
            _, checks, _, _, _ = do.punctured_rows(k, m, present)
            buf = clean.clone()
            keys = tde.inject_counting(torch, buf, checks, 0, length, 8 * c)
            t = min(radius, c // 2)
            a, b, va, vb = tde.blame(torch, do.error_table(k, m, t, present), keys)
            plain = {i: clean[i, :length] for i in lost if i < k}
            got = check_decode(torch, enc, buf, 0, length, k, m, present, radius, a, b, va, vb, keys != 0, plain,
                               null_parity=n_case % 2 == 1, rebuild=True)
            assert got["damaged_columns"] == length - 1
            assert got["uncorrectable_columns"] == length - 1 - (0 if t == 0 else (k + c) * 255), lost


@pytest.mark.gpu
def test_decode_rs_10_4_three_and_four_lost(cuda, swec):
    """c = 1: every damaged column is uncorrectable and the data are those of a data-only reconstruct on the shards as
    found; c = 0: nothing is checked (columns = 0, no ranges, no locate kernel) and the data are those of a data-only
    reconstruct, damage included."""
    torch = cuda
    k, m, length = 10, 4, 256
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    clean = tde.tiled(torch, k, m, length, seed=34)
    unchecked = {"columns": 0, "damaged_columns": 0, "uncorrectable_columns": 0, "first_uncorrectable": -1,
                 "last_uncorrectable": -1, "shards": {}, "ranges": [], "n_ranges": 0}
    for f in (3, 4):
        for n_case, lost in enumerate(itertools.combinations(range(k + m), f)):
            present = tde.mask(k + m, lost)
            info, checks, _, _, _ = do.punctured_rows(k, m, present)
            buf = clean.clone()
            if checks:
                keys = tde.inject_counting(torch, buf, checks, 0, length, 8)
                a, b, va, vb = tde.blame(torch, do.error_table(k, m, 0, present), keys)
                assert not (a >= 0).any()
            else:                                   # damage an information shard: nothing can see it
                keys = torch.arange(length, device=tde.DEV) & 255
                buf[info[0], :length] ^= keys.to(torch.uint8)
            fill_lost(buf, k, lost)
            plain = buf.clone()
            enc.reconstruct_device(tde.ptrs(plain, 0), [int(x) for x in present], length, data_only=True)
            null_parity = n_case % 2 == 1
            if checks:
                got = check_decode(torch, enc, buf, 0, length, k, m, present, 1, a, b, va, vb, keys != 0,
                                   {i: clean[i, :length] for i in lost if i < k}, null_parity=null_parity)
                assert got["uncorrectable_columns"] == got["damaged_columns"] == length - 1, lost
            else:                                   # no check shard: no locate kernel at all
                before = buf.clone()
                got = enc.decode_data_checked_device(decode_ptrs(buf, 0, k, lost, null_parity),
                                                     [int(x) for x in present], length, radius=1)
                assert got == unchecked, lost
                assert torch.equal(buf[k:], before[k:]), lost
            torch.cuda.synchronize()
            assert torch.equal(buf[:k], plain[:k]), lost


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("k,m,lost", [(k, m, ()) for k, m in tde.SMALL] + [(1, 3, (0,))])
def test_decode_every_syndrome_of_m_2_and_3(cuda, swec, k, m, lost, shift):
    """Radius 1: column x carries syndrome x mod 2^(8c), the 7 columns past 2^(8c) repeat syndromes 0..6 in the tail;
    at offset 3 every stream goes through the byte loop.  RS(1,3) with shard 0 lost decodes from parity shard 1."""
    torch = cuda
    present = tde.mask(k + m, lost)
    _, checks, _, _, _ = do.punctured_rows(k, m, present)
    c = len(checks)
    length = (1 << (8 * c)) + 7
    buf = tde.tiled(torch, k, m, length, seed=k * 10 + m + len(lost), shift=shift)
    plain = {i: buf[i, shift:shift + length].clone() for i in lost if i < k}
    keys = tde.inject_counting(torch, buf, checks, shift, length, 8 * c)
    a, b, va, vb = tde.blame(torch, do.error_table(k, m, 1, present), keys)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    got = check_decode(torch, enc, buf, shift, length, k, m, present, 1, a, b, va, vb, keys != 0, plain,
                       null_parity=shift == 3)
    assert got["damaged_columns"] == length - 2 and len(got["shards"]) == k + c
    assert got["uncorrectable_columns"] == length - 2 - (k + c) * 255 - 6


@pytest.mark.gpu
@pytest.mark.parametrize("lost", [(), (3,), (9,)])
def test_decode_rs_8_6_radius_2_every_pattern(cuda, swec, lost):
    """Any c at radius 2: every pattern of 1 or 2 wrong positions with every value (5,920,845 with nothing lost, then
    2^24 random syndromes; 5,075,265 with data shard 3 or parity shard 9 lost)."""
    torch = cuda
    k, m, radius = 8, 6, 2
    present = tde.mask(k + m, lost)
    _, checks, _, _, _ = do.punctured_rows(k, m, present)
    c = len(checks)
    table = do.error_table(k, m, radius, present)
    syn = table[1]
    if not lost:
        rng = np.random.default_rng(860)
        syn = np.concatenate([syn, rng.integers(0, 256, (1 << 24, c), dtype=np.uint8)])
    length = len(syn)
    n_table = len(table[0])
    assert n_table == (k + c) * 255 + (k + c) * (k + c - 1) // 2 * 255 * 255
    buf = tde.tiled(torch, k, m, length, seed=861 + len(lost))
    plain = {i: buf[i, :length].clone() for i in lost if i < k}
    syn_gpu = torch.from_numpy(syn).to(tde.DEV)
    for i, row in enumerate(checks):
        buf[row, :length] ^= syn_gpu[:, i]
    keys = tde.key_of(torch, syn_gpu)
    a, b, va, vb = tde.blame(torch, table, keys)
    assert (a[:n_table].cpu().numpy() == table[2]).all() and (b[:n_table].cpu().numpy() == table[3]).all()
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    got = check_decode(torch, enc, buf, 0, length, k, m, present, radius, a, b, va, vb, keys != 0, plain,
                       null_parity=True)
    assert got["damaged_columns"] == length - int((keys == 0).sum())
    assert len(got["shards"]) == k + c and got["uncorrectable_columns"] == length - int((a >= 0).sum()) - int(
        (keys == 0).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,lost", [(5, 5, ()), (8, 6, tde.RS86_LOST)])
def test_decode_every_pattern_with_one_syndrome_byte_cleared(cuda, swec, k, m, lost):
    """Every syndrome of the radius-2 table with each byte cleared in turn (c = 5): 14,643,375 columns for RS(5,5),
    25,376,325 for RS(8,6) with shard 3 lost.  One with 3 .. c-2 non-zero bytes is uncorrectable."""
    torch = cuda
    present = tde.mask(k + m, lost)
    _, checks, _, _, _ = do.punctured_rows(k, m, present)
    c = len(checks)
    table = do.error_table(k, m, 2, present)
    syn = np.repeat(table[1], c, axis=0)
    syn[np.arange(len(syn)), np.tile(np.arange(c), len(table[1]))] = 0
    length = len(syn)
    buf = tde.tiled(torch, k, m, length, seed=k * 10 + m + 1)
    plain = {i: buf[i, :length].clone() for i in lost if i < k}
    syn_gpu = torch.from_numpy(syn).to(tde.DEV)
    for i, row in enumerate(checks):
        buf[row, :length] ^= syn_gpu[:, i]
    keys = tde.key_of(torch, syn_gpu)
    a, b, va, vb = tde.blame(torch, table, keys)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    got = check_decode(torch, enc, buf, 0, length, k, m, present, 2, a, b, va, vb, keys != 0, plain)
    weight = (syn_gpu != 0).sum(dim=1)
    assert got["uncorrectable_columns"] >= int(((weight >= 3) & (weight <= c - 2)).sum()) > 0


@pytest.mark.gpu
def test_decode_across_the_piece_boundary(cuda, swec):
    """RS(10,4) with shard 2 lost, 2^28 + 4,103 columns: the call works in pieces of 256 MiB.  Column x < 2^28 carries
    check syndrome x mod 2^24; the columns past the boundary carry every correctable syndrome once, then uncorrectable
    ones, so every shard's last column, the last uncorrectable one, their page ranges and the corrections all lie in
    the second piece."""
    torch = cuda
    if tde.free_bytes(torch) < 16 * tde.GIB:
        pytest.skip("needs 16 GiB of free device memory")
    k, m, lost = 10, 4, (2,)
    piece = 1 << 28
    length = piece + 4103
    present = tde.mask(k + m, lost)
    _, checks, _, _, _ = do.punctured_rows(k, m, present)
    table = do.error_table(k, m, 1, present)
    buf = tde.tiled(torch, k, m, length, seed=228)
    plain = {2: buf[2, :length].clone()}
    keys = torch.arange(length, dtype=torch.int64, device=tde.DEV) & ((1 << 24) - 1)
    n_table = len(table[0])
    keys[piece:piece + n_table] = tde.key_of(torch, torch.from_numpy(table[1]).to(tde.DEV))
    inject_keys(torch, buf, checks, 0, keys)
    a, b, va, vb = tde.blame(torch, table, keys)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    got = check_decode(torch, enc, buf, 0, length, k, m, present, 1, a, b, va, vb, keys != 0, plain)
    assert len(got["shards"]) == 13 and all(last >= piece for _, _, last in got["shards"].values())
    assert got["last_uncorrectable"] >= piece + n_table
    assert any(off >= piece for sid, off, _ in got["ranges"] if sid >= 0)


# ------------------------------------------------------------------------------------------ GPU: the guarantee


def loss_sets(k, m, rng):
    """nothing, one data shard, one parity shard, m-2 and m-4 shards of both kinds (where there are that many)"""
    out = [(), (int(rng.integers(k)),), (k + int(rng.integers(m)),)]
    for f in (m - 2, m - 4):
        if f >= 1:
            nd = min(k, max(1, f // 2))
            data = rng.choice(k, size=nd, replace=False)
            parity = k + rng.choice(m, size=f - nd, replace=False)
            out.append(tuple(sorted(int(i) for i in np.concatenate([data, parity]))))
    if (k, m) == (16, 16):
        out.append(tuple(range(2, 16)))              # c = 2 with the widest position map
    return list(dict.fromkeys(out))


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("k,m", tde.SHAPES)
def test_decode_guarantee_against_injected_damage(cuda, swec, k, m, shift):
    """20,007 columns with w = 1 .. c-t wrong present shards: w <= t, every data byte is the true one; t < w, the
    column is uncorrectable and its data bytes are those of a plain data-only reconstruct from the shards as found.
    Present parity is never written."""
    torch = cuda
    n, length = k + m, 20_007
    clean = np.stack(tde.random_set(k, m, length, seed=n * 1000 + m + 7))
    clean_gpu = torch.from_numpy(clean).to(tde.DEV)
    mul = tde.gmul_table(torch)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    rng = np.random.default_rng(n * 100 + m + shift)
    for n_case, lost in enumerate(loss_sets(k, m, rng)):
        present = tde.mask(n, lost)
        info, checks, _, _, r = do.punctured_rows(k, m, present)
        c = len(checks)
        for radius in (0, 1, 2):
            t = min(radius, c // 2)
            err, w = tde.random_damage(n, length, c - t, rng, ids=info + checks)
            found = torch.from_numpy(clean ^ err.T).to(tde.DEV)
            buf = tde.buffer(torch, n, length, shift)
            buf[:, shift:shift + length] = found
            fill_lost(buf, k, lost)
            within = torch.from_numpy(w <= t).to(tde.DEV)
            a, b = tde.first_two(torch, err)
            ida, idb = torch.where(within, a, -1), torch.where(within, b, -1)
            want = tde.without_ok(do.dense_report(ida, idb, torch.ones(length, dtype=torch.bool, device=tde.DEV),
                                                  n))
            exp = buf.clone()
            for row, i in enumerate(lost):
                if i < k:                          # plain rebuild from the information set as found
                    plain = torch.zeros(length, dtype=torch.uint8, device=tde.DEV)
                    for j, src in enumerate(info):
                        plain ^= tde.gmul(mul, int(r[row][j]), found[src])
                    exp[i, shift:shift + length] = torch.where(within, clean_gpu[i], plain)
            for i in range(k):
                if present[i]:
                    exp[i, shift:shift + length] = torch.where(within, clean_gpu[i], found[i])
            got = enc.decode_data_checked_device(decode_ptrs(buf, shift, k, lost, (n_case + radius) % 2 == 1),
                                                 [int(x) for x in present], length, radius=radius,
                                                 max_ranges=tde.MAX_RANGES)
            assert got == want, (lost, radius)
            assert want["uncorrectable_columns"] == int((w > t).sum()), (lost, radius)
            assert torch.equal(buf, exp), (lost, radius)


# ------------------------------------------------------------------------------------------ GPU: file level


@pytest.mark.gpu
@pytest.mark.parametrize("lost", [(5, 13), (5, 27)])
def test_file_level_decode_at_rs_20_12_radius_2(cuda, swec, oracle, tmp_path, monkeypatch, lost):
    """write_dat_file_checked with 100-byte small and 10000-byte large blocks in 4 KiB slots writes the device-level
    decode un-striped by the copy plan, and reports what the device call reports; a missing parity shard is not
    rebuilt.  With one column of 3 wrong shards, ec_shards_to_volume_checked raises SWEC_ERR_UNCORRECTABLE with the
    device call's report and leaves neither .dat nor .idx."""
    torch = cuda
    ec = swec.erasure_coding
    monkeypatch.setenv("SWEC_FILE_CHUNK", "4096")
    k, m, t = 20, 12, 2
    n = k + m
    present = tde.mask(n, lost)
    ids = [i for i in range(n) if present[i]]
    enc = ec.Encoder(k, m, device=0)

    def device_decode(shards, length):
        buf = tde.buffer(torch, n, length, 0)
        for i in ids:
            buf[i, :length] = torch.from_numpy(shards[i][:length]).to(tde.DEV)
        fill_lost(buf, k, lost)
        rep = enc.decode_data_checked_device(decode_ptrs(buf, 0, k, lost, True), [int(x) for x in present], length,
                                             radius=t)
        return buf, rep

    dat_size = 3 * k * 10000 + 57 * k * 100 + 3 * 100 + 37
    base, dat, clean = tcd._small_block_set(oracle, tmp_path, k, m, dat_size, seed=2020 + lost[1])
    size = len(clean[0])
    rng = np.random.default_rng(2021 + lost[1])
    err, _ = tde.random_damage(n, size, t, rng, ids=ids)
    err[rng.random(size) < 0.5] = 0
    damaged = [s ^ e for s, e in zip(clean, err.T)]
    tcr.write_set(base, damaged)
    tcr.remove(base, lost)
    names = [base + ".ec%02d" % i if present[i] else None for i in range(n)]
    res = ec.write_dat_file_checked(str(tmp_path / "out"), dat_size, names, data_shards=k, parity_shards=m,
                                    large_block=10000, small_block=100, radius=t)
    cols = res["columns"]
    assert cols == 3 * 10000 + 57 * 100 + 100 and res["ok"] and res["damaged_columns"] > 0
    buf, dev = device_decode(damaged, cols)
    assert {key: v for key, v in res.items() if key not in ("dat_file_size", "ok")} == dev
    out = torch.zeros(dat_size, dtype=torch.uint8, device=tde.DEV)
    enc.write_dat_device([buf[i].data_ptr() for i in range(k)], dat_size, out.data_ptr(), large_block=10000,
                         small_block=100)
    torch.cuda.synchronize()
    written = np.fromfile(str(tmp_path / "out.dat"), dtype=np.uint8)
    assert (written == out.cpu().numpy()).all() and (written == dat).all()
    assert not any(os.path.exists(base + ".ec%02d" % i) for i in lost)

    dat2, idx2 = tcd.needle_volume(seed=2022 + lost[1], needles=150)
    (tmp_path / "v").mkdir()
    vbase, vclean = tcd.lay_down(oracle, tmp_path / "v", dat2, idx2, k=k, m=m)
    vsize = len(vclean[0])
    err, _ = tde.random_damage(n, vsize, t, rng, ids=ids)
    err[rng.random(vsize) < 0.9] = 0
    x0 = 777
    err[x0] = 0
    err[x0, rng.choice(ids, 3, replace=False)] = rng.integers(1, 256, 3)
    vdamaged = [s ^ e for s, e in zip(vclean, err.T)]
    tcr.write_set(vbase, vdamaged)
    tcr.remove(vbase, lost)
    with pytest.raises(swec.SwecError) as e:
        ec.ec_shards_to_volume_checked(vbase, radius=t)
    assert e.value.name == "SWEC_ERR_UNCORRECTABLE"
    rep = e.value.report
    assert rep["uncorrectable_columns"] == 1 and rep["first_uncorrectable"] == rep["last_uncorrectable"] == x0
    assert rep == device_decode(vdamaged, rep["columns"])[1]
    assert tcd.no_outputs(vbase)
    assert not any(os.path.exists(vbase + ".ec%02d" % i) for i in lost)


# ------------------------------------------------------------------------------------------ GPU: the ledger


# The instantiation a call runs depends on its mode and on m (locate, correct) or c (rebuild, decode) alone, so one small
# call per sweep configuration names it.  torch.profiler runs in a process of its own: CUPTI's state outlives a
# profiling session, and the profiler in the pytest process would change what test_kernel_variants.py records later.

# (label, k, m, lost, mode, radius, the instantiations the call must run: none for a decode with no check shard)
NAME_CASES = [("RS(10,4) nothing lost", 10, 4, (), "decode", 2, {decode_id(4)}),
              ("RS(10,4) one data lost", 10, 4, (3,), "decode", 2, {decode_id(3)}),
              ("RS(10,4) one parity lost", 10, 4, (12,), "decode", 1, {decode_id(3)}),
              ("RS(10,4) two lost", 10, 4, (0, 11), "decode", 1, {decode_id(2)}),
              ("RS(10,4) three lost", 10, 4, (0, 1, 2), "decode", 1, {decode_id(1)}),
              ("RS(10,4) four lost", 10, 4, (0, 1, 2, 3), "decode", 1, set()),
              ("RS(10,4) shard 2 lost", 10, 4, (2,), "decode", 1, {decode_id(3)}),
              ("RS(3,2)", 3, 2, (), "decode", 1, {decode_id(2)}), ("RS(6,3)", 6, 3, (), "decode", 1, {decode_id(3)}),
              ("RS(1,3) shard 0 lost", 1, 3, (0,), "decode", 1, {decode_id(2)}),
              ("RS(8,6) nothing lost", 8, 6, (), "decode", 2, {decode_id(6)}),
              ("RS(8,6) shard 9 lost", 8, 6, (9,), "decode", 2, {decode_id(5)}),
              ("RS(5,5)", 5, 5, (), "decode", 2, {decode_id(5)}),
              ("RS(28,4)", 28, 4, (), "decode", 2, {decode_id(4)}),
              ("RS(16,16) 14 data lost", 16, 16, tuple(range(2, 16)), "decode", 2, {decode_id(2)}),
              ("locate m = 4", 10, 4, (), "locate", 1, {(4, LOCATE)}), ("locate m = 3", 6, 3, (), "locate", 1, {(0, LOCATE)}),
              ("correct m = 4", 10, 4, (), "correct", 1, {(4, CORRECT)}),
              ("correct m = 3", 6, 3, (), "correct", 1, {(0, CORRECT)}),
              ("rebuild c = 3", 10, 4, (3,), "rebuild", 1, {rebuild_id(3)}),
              ("rebuild c = 2", 10, 4, (0, 11), "rebuild", 1, {rebuild_id(2)})]


def _names_child():
    """Runs in a fresh process: one call of 4,099 columns per NAME_CASES entry, with one wrong byte in the lowest
    present shard, under torch.profiler.  Prints RESULT <json>: per label, the report and the sorted (MT, MODE) that ran, or
    None when the profiler recorded no kernel at all."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    import seaweedfs_b200.erasure_coding as ec
    out = {}
    length = 4099
    for label, k, m, lost, mode, radius, _ in NAME_CASES:
        n = k + m
        shards = tde.random_set(k, m, length, seed=n + len(lost))
        bad = next(i for i in range(n) if i not in lost)
        shards[bad][1000] ^= 0x40
        present = tde.mask(n, lost)
        buf = torch.zeros((n, length + 29), dtype=torch.uint8, device="cuda")
        buf[:, :length] = torch.from_numpy(np.stack(shards)).cuda()
        fill_lost(buf, k, lost)
        p = [buf[i].data_ptr() for i in range(n)]
        enc = ec.Encoder(k, m, device=0)
        call = {"locate": lambda: enc.locate_damage_device(p, length, radius=radius),
                "correct": lambda: enc.correct_damage_device(p, length, radius=radius),
                "rebuild": lambda: enc.reconstruct_checked_device(p, present, length, radius=radius),
                "decode": lambda: enc.decode_data_checked_device(p, [int(x) for x in present], length, radius=radius)}
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            rep = call[mode]()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
        ids = sorted({locate_id(x) for x in names} - {None}) if names else None
        fixed = int(buf[bad, 1000].item()) == int(shards[bad][1000] ^ 0x40)
        out[label] = {"ids": ids, "damaged": rep["damaged_columns"], "shards": sorted(rep["shards"]), "bad": bad,
                      "fixed": fixed}
        enc.close()
    print("RESULT " + json.dumps(out))


@pytest.mark.gpu
def test_every_locate_instantiation_runs_by_name(cuda, swec):
    """Every instantiation of LEDGER runs, and every sweep configuration above runs the one its mode and c select."""
    assert set().union(*(want for *_, want in NAME_CASES)) == LEDGER
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{tcd.ROOT!r}, {here!r}]; "
            "import test_decode_exhaustive as t; t._names_child()")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(next(ln for ln in r.stdout.splitlines() if ln.startswith("RESULT "))[7:])
    for label, k, m, lost, mode, radius, want in NAME_CASES:
        res = got[label]
        if res["ids"] is None:
            tkv.no_names(label)
        else:
            assert {tuple(i) for i in res["ids"]} == want, (label, res["ids"], sorted(want))
        c = m - len(lost)
        t = radius if mode in ("locate", "correct") else min(radius, c // 2)
        if c == 0:
            assert res["damaged"] == 0, label                     # nothing to check the shards against
        else:
            assert res["damaged"] == 1 and res["shards"] == ([res["bad"]] if t else []), (label, res)
        # present shards are written by correct, and by decode where a data shard is decoded within the radius
        assert res["fixed"] == (mode == "correct" or (mode == "decode" and t > 0 and res["bad"] < k)), (label, res)
