"""The damage decoder (decode_column in seaweedfs_b200/csrc/damage.cu) at every syndrome of the small codes, and the
include/swec.h guarantee against injected damage on every code shape the encoder accepts up to k + m = 32.

The decoder's answer depends on a column's syndrome alone, so the input space of a small code can be enumerated: column
x of a shard set carries a chosen syndrome when the stored parity (or the stored check shards) of a tiled random codeword
is XORed with the syndrome's bytes.  The expected report and bytes follow from the exhaustive error table of
tests/damage_oracle.py (error_table, any m), looked up on the GPU.  Every sweep compares the whole report and every byte
of every shard buffer after the call.

cpu: the any-m oracle equals damage_oracle.locate and the correction oracle of test_damage_repair.py (radius 1 on every
shape below with m <= 8, radius 2 where k + m <= 16) and the checked-rebuild oracle of test_checked_rebuild.py; the
tables of every sweep are collision-free (MDS within the radius); dense_report equals damage_oracle.report.
gpu, syndrome sweeps (locate and correct unless named):
  - m = 2 and 3, radius 1, every non-zero syndrome: RS(3,2), RS(30,2) (65,535 each), RS(1,3), RS(6,3), RS(29,3)
    (16,777,215 each); once aligned with 7 more columns (the tail), once at a pointer offset of 3 (the byte path);
  - RS(10,4), radius 1 and 2: all 4,294,967,295 non-zero syndromes, 16 calls of 2^28 columns each, per radius and call;
  - checked rebuild of RS(10,4), radius 0, 1 and 2: each of the 14 single losses (c = 3) at all 16,777,215 non-zero
    check syndromes, and each of the 91 double losses (c = 2) at all 65,535;
  - checked rebuild of RS(8,6) with shard 3 lost (c = 5, radius 2): all 5,075,265 patterns of 1 or 2 wrong present
    shards with every value, then 16,777,216 random syndromes;
  - radius 2, c = 5: every syndrome of the table with each of its bytes cleared in turn, next to a decodable one:
    RS(5,5) locate and correct (14,643,375 columns), RS(8,6) with shard 3 lost, checked rebuild (25,376,325).
gpu, the guarantee on RS(1,2), RS(4,2), RS(5,5), RS(1,31), RS(24,8), RS(28,4), RS(20,12), RS(16,16) at radius t = 1 and 2
(2t <= m), checked against the injected damage, not an oracle:
  - 30,007 columns with w = 1 .. m-t wrong shards drawn from all shards, random non-zero values, aligned and at offset 3:
    w <= t blamed exactly and corrected to the clean set; t < w uncorrectable, nothing blamed, every byte left as it was;
  - every pattern within the radius over every shard and shard pair: every value up to m = 8 (n·255 + C(n,2)·255²
    columns, 32,248,560 for k + m = 32), 255 random value pairs per shard pair past m = 8;
  - checked rebuild with f = 1, m-2 and m-4 shards lost (c = m - f), radius 0, 1 and 2, 20,007 columns with 1 .. c-t
    wrong present shards: blamed and rebuilt right, or uncorrectable and rebuilt as plain rebuild does;
  - RS(20,12) at radius 2 through ECContext: locate, repair, and checked rebuild with 2 shards lost (42 streams a slot)
    report what the device-level calls report, and write what they write."""
import itertools
import os
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import damage_oracle as do  # noqa: E402
import test_checked_rebuild as tcr  # noqa: E402
import test_damage_repair as tdr  # noqa: E402

from oracle import rs_numpy as rn  # noqa: E402

GIB = 1 << 30
SLICE_BITS = 28
PERIOD = 4093          # the base codeword set repeats every PERIOD columns (a prime: no vector or page repeats it)
MAX_RANGES = 1 << 20   # room for every range of a sweep
SMALL = [(3, 2), (30, 2), (1, 3), (6, 3), (29, 3)]
SHAPES = [(1, 2), (4, 2), (5, 5), (1, 31), (24, 8), (28, 4), (20, 12), (16, 16)]
RS86_LOST = (3,)
DEV = "cuda"           # where the sweeps build their inputs and expectations ("cpu" runs the helpers without a GPU)


def random_set(k, m, length, seed):
    rng = np.random.default_rng(seed)
    data = [rng.integers(0, 256, length, dtype=np.uint8) for _ in range(k)]
    return data + rn.encode(k, m, data)


def mask(n, lost):
    return tuple(i not in lost for i in range(n))


def radii(m):
    return [t for t in (1, 2) if 2 * t <= m]


# ------------------------------------------------------------------------------------------ CPU


def fuzz(k, m, length, most, seed, present=None):
    """A random set with 1..most random present shards wrong in a third of the columns."""
    rng = np.random.default_rng(seed)
    shards = random_set(k, m, length, seed)
    ids = [i for i in range(k + m) if present is None or present[i]]
    for c in rng.choice(length, size=length // 3, replace=False):
        for sid in rng.choice(ids, size=min(len(ids), int(rng.integers(1, most + 1))), replace=False):
            shards[int(sid)][c] ^= np.uint8(rng.integers(1, 256))
    return shards


AGREE = sorted({s for s in SMALL + SHAPES + [(10, 4), (8, 6)] if s[1] <= 8})


@pytest.mark.parametrize("k,m", AGREE)
def test_any_m_oracle_agrees_with_the_uint64_oracles(k, m):
    n = k + m
    for radius in [t for t in radii(m) if t == 1 or n <= 16]:
        shards = fuzz(k, m, 3001, 2 * radius + 1, seed=n * 10 + radius)
        cols, a, b, va, vb, ids = do.decode_columns(shards, k, m, radius)
        ida, idb = (np.where(p >= 0, ids[np.maximum(p, 0)], -1) for p in (a, b))
        assert do.report(3001, n, cols, ida, idb) == do.locate(shards, k, m, radius), radius
        fixed = [s.copy() for s in shards]
        for p, v in ((ida, va), (idb, vb)):
            for sid in range(n):
                fixed[sid][cols[p == sid]] ^= v[p == sid]
        assert tdr.same(fixed, tdr.correct(shards, k, m, radius)), radius


@pytest.mark.parametrize("k,m,lost,radius", [(10, 4, (4,), 1), (10, 4, (0, 11), 2), (8, 6, RS86_LOST, 2)])
def test_any_m_oracle_agrees_with_the_checked_rebuild_oracle(k, m, lost, radius):
    present = mask(k + m, lost)
    shards = fuzz(k, m, 2001, 3, seed=len(lost) * 7 + m, present=present)
    c = m - len(lost)
    cols, a, b, va, vb, ids = do.decode_columns(shards, k, m, min(radius, c // 2), present)
    ida, idb = (np.where(p >= 0, ids[np.maximum(p, 0)], -1) for p in (a, b))
    _, want = tcr.checked_rebuild(shards, k, m, present, radius)
    assert do.report(2001, k + m, cols, ida, idb) == {**want, "ok": len(cols) == 0}


def sweep_tables():
    """(k, m, radius, presence mask or None) of every table a GPU sweep looks its syndromes up in."""
    out = [(k, m, 1, None) for k, m in SMALL] + [(10, 4, 1, None), (10, 4, 2, None)]
    for f in (1, 2):
        for lost in itertools.combinations(range(14), f):
            out += [(10, 4, 1, mask(14, lost))]
    return out + [(8, 6, 2, mask(14, RS86_LOST))]


def test_every_sweep_table_is_collision_free():
    """error_table asserts that no two patterns share a syndrome; the sizes say that every pattern is in it."""
    for k, m, radius, present in sweep_tables():
        n = k + (m if present is None else sum(present) - k)
        keys = do.error_table(k, m, radius, present)[0]
        assert len(keys) == n * 255 + (n * (n - 1) // 2 * 255 * 255 if radius == 2 else 0), (k, m, radius, present)
    assert len(sweep_tables()) == 5 + 2 + 14 + 91 + 1


def test_dense_report_equals_report():
    import torch
    rng = np.random.default_rng(7)
    for length, n in ((1, 3), (4096, 14), (3 * 4096 + 5, 14), (40_000, 32)):
        for density in (0.0, 0.001, 0.3, 1.0):
            cols = np.flatnonzero(rng.random(length) < density)
            a = rng.integers(-1, n, len(cols))
            b = np.where((a >= 0) & (rng.random(len(cols)) < 0.3), rng.integers(0, n, len(cols)), -1)
            b = np.where(b == a, -1, b)
            da, db = np.full(length, -1), np.full(length, -1)
            da[cols], db[cols] = a, b
            damaged = np.zeros(length, dtype=bool)
            damaged[cols] = True
            got = do.dense_report(torch.from_numpy(da), torch.from_numpy(db), torch.from_numpy(damaged), n)
            assert got == do.report(length, n, cols, a, b), (length, n, density)


# ------------------------------------------------------------------------------------------ GPU helpers


def without_ok(rep):
    return {key: v for key, v in rep.items() if key != "ok"}


def buffer(torch, n, length, shift):
    """(n, width) zeros on the GPU; row i holds shard i at columns [shift, shift + length), rows 16-byte aligned."""
    return torch.zeros((n, (shift + length + 31) // 16 * 16), dtype=torch.uint8, device=DEV)


def ptrs(buf, shift):
    return [buf[i].data_ptr() + shift for i in range(len(buf))]


def tiled(torch, k, m, length, seed, shift=0):
    """A random codeword set of PERIOD columns, repeated over `length` columns of a buffer."""
    base = torch.from_numpy(np.stack(random_set(k, m, PERIOD, seed))).to(DEV)
    assert base.any(dim=1).all()
    buf = buffer(torch, k + m, length, shift)
    reps = -(-length // PERIOD)
    for i in range(k + m):
        buf[i, shift:shift + length] = base[i].repeat(reps)[:length]
    return buf


def inject_counting(torch, buf, rows, shift, length, bits, lo=0):
    """XOR syndrome lo + (x mod 2^bits) into the `rows` (byte i into rows[i]) at column x; returns the keys (int64)."""
    keys = (torch.arange(length, dtype=torch.int64, device=DEV) & ((1 << bits) - 1)) | lo
    for i, r in enumerate(rows):
        buf[r, shift:shift + length] ^= ((keys >> (8 * i)) & 255).to(torch.uint8)
    return keys


def key_of(torch, syn):
    """damage_oracle._keys on the GPU: syndrome bytes (N, c) -> int64, byte i at bits 8i."""
    key = torch.zeros(len(syn), dtype=torch.int64, device=syn.device)
    for i in range(syn.shape[1]):
        key |= syn[:, i].to(torch.int64) << (8 * i)
    return key


def blame(torch, table, keys, chunk=1 << 26):
    """(a, b, va, vb) of every column from its syndrome key, looked up in an error_table on the GPU."""
    _, syn, *vals = table
    out = [torch.full((len(keys),), fill, dtype=dt, device=DEV)
           for fill, dt in ((-1, torch.int8), (-1, torch.int8), (0, torch.uint8), (0, torch.uint8))]
    if not len(syn):
        return out
    tk, order = torch.sort(key_of(torch, torch.from_numpy(syn).to(DEV)))
    vals = [torch.from_numpy(v).to(DEV)[order].to(o.dtype) for v, o in zip(vals, out)]
    for lo in range(0, len(keys), chunk):
        q = keys[lo:lo + chunk]
        pos = torch.searchsorted(tk, q).clamp_(max=len(tk) - 1)
        hit = tk[pos] == q
        for o, v in zip(out, vals):
            o[lo:lo + chunk] = torch.where(hit, v[pos], o[lo:lo + chunk])
    return out


def to_ids(torch, ids, p):
    """positions (-1: none) -> shard ids"""
    t = torch.tensor([-1] + list(ids), dtype=torch.int8, device=DEV)
    return t[p.long() + 1]


def gmul_table(torch):
    return torch.from_numpy(rn.MUL).to(DEV)


def gmul(mul, coef, v):
    """coef·v per byte (coef: a tensor of coefficients, or one int)"""
    if isinstance(coef, int):
        return mul[coef][v.long()]
    return mul[coef.long(), v.long()]


def undo_correction(torch, buf, shift, a, b, va, vb, ids):
    """XOR every column's expected correction back out of the shard rows (ids[p] is position p's row)."""
    length = len(a)
    for p, sid in enumerate(ids):
        buf[sid, shift:shift + length] ^= torch.where(a == p, va, 0) ^ torch.where(b == p, vb, 0)


def check_locate_and_correct(torch, enc, buf, shift, length, radius, a, b, va, vb, damaged, max_ranges=MAX_RANGES):
    """Locate leaves every byte as it was, correct writes exactly the expected corrections; both report `want`."""
    n = len(buf)
    want = without_ok(do.dense_report(a, b, damaged, n))
    before = buf.clone()
    assert enc.locate_damage_device(ptrs(buf, shift), length, radius=radius, max_ranges=max_ranges) == want
    assert torch.equal(buf, before)
    assert enc.correct_damage_device(ptrs(buf, shift), length, radius=radius, max_ranges=max_ranges) == want
    undo_correction(torch, buf, shift, a, b, va, vb, range(n))
    assert torch.equal(buf, before)
    return want


# ------------------------------------------------------------------------------------------ GPU: syndrome sweeps


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("k,m", SMALL)
def test_every_syndrome_of_m_2_and_3(cuda, swec, k, m, shift):
    """Column x carries syndrome x mod 2^(8m); the 7 columns past 2^(8m) repeat syndromes 0..6 in the tail."""
    torch = cuda
    length = (1 << (8 * m)) + 7
    buf = tiled(torch, k, m, length, seed=k * 10 + m, shift=shift)
    keys = inject_counting(torch, buf, range(k, k + m), shift, length, 8 * m)
    a, b, va, vb = blame(torch, do.error_table(k, m, 1), keys)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    want = check_locate_and_correct(torch, enc, buf, shift, length, 1, a, b, va, vb, keys != 0)
    # two clean columns (syndrome 0); blamed: every single-shard syndrome, and syndromes 1..6 again in the tail
    assert want["damaged_columns"] == length - 2 and len(want["shards"]) == k + m
    assert want["uncorrectable_columns"] == length - 2 - (k + m) * 255 - 6


def free_bytes(torch):
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [1, 2])
def test_every_syndrome_of_rs_10_4(cuda, swec, radius):
    """All 2^32 syndromes of the production code, 2^28 columns a call: column x of slice s carries s·2^28 + x."""
    torch = cuda
    if free_bytes(torch) < 16 * GIB:
        pytest.skip("needs 16 GiB of free device memory")
    k, m = 10, 4
    n_slice = 1 << SLICE_BITS
    table = do.error_table(k, m, radius)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    clean = tiled(torch, k, m, n_slice, seed=104)
    blamed = uncorrectable = 0
    times = []
    for s in range(1 << (32 - SLICE_BITS)):
        t0 = time.perf_counter()
        buf = clean.clone()
        keys = inject_counting(torch, buf, range(k, k + m), 0, n_slice, SLICE_BITS, lo=s << SLICE_BITS)
        a, b, va, vb = blame(torch, table, keys)
        want = check_locate_and_correct(torch, enc, buf, 0, n_slice, radius, a, b, va, vb, keys != 0)
        blamed += int((a >= 0).sum())
        uncorrectable += want["uncorrectable_columns"]
        del buf, keys, a, b, va, vb
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    assert blamed == len(table[0]) and blamed + uncorrectable == (1 << 32) - 1
    print(f"\nRS(10,4) radius {radius}: 16 slices of 2^28 columns, locate + correct + expected, "
          f"{min(times):.2f} .. {max(times):.2f} s a slice, {sum(times):.1f} s in all")


def check_rebuild(torch, enc, buf, shift, length, k, m, present, radius, a, b, va, vb, damaged, want_lost):
    """The checked rebuild reports the blame (positions a, b) and writes want_lost + the images of the information
    errors it takes out into the lost rows; present rows stay as they were."""
    info, checks, lost, _, r = do.punctured_rows(k, m, tuple(present))
    ids = info + checks
    want = without_ok(do.dense_report(to_ids(torch, ids, a), to_ids(torch, ids, b), damaged, k + m))
    mul = gmul_table(torch)
    for i in lost:
        buf[i].zero_()
    before = buf.clone()
    got = enc.reconstruct_checked_device(ptrs(buf, shift), present, length, radius=radius, max_ranges=MAX_RANGES)
    assert got == want, radius
    for row, i in enumerate(lost):
        coef = torch.zeros(k + len(checks) + 1, dtype=torch.uint8, device=DEV)   # by position + 1; 0 for a check
        coef[1:k + 1] = torch.from_numpy(r[row]).to(DEV)
        out = buf[i, shift:shift + length]
        out ^= want_lost[row] ^ gmul(mul, coef[a.long() + 1], va) ^ gmul(mul, coef[b.long() + 1], vb)
    assert torch.equal(buf, before), radius
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("radius", [0, 1, 2])
def test_checked_rebuild_every_check_syndrome_of_rs_10_4(cuda, swec, radius):
    """14 single losses x 2^24 check syndromes (c = 3), 91 double losses x 2^16 (c = 2); radius 2 clamps to 1."""
    torch = cuda
    k, m = 10, 4
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    for f in (1, 2):
        c = m - f
        length = 1 << (8 * c)
        clean = tiled(torch, k, m, length, seed=f)
        for lost in itertools.combinations(range(k + m), f):
            present = mask(k + m, lost)
            info, checks, _, _, _ = do.punctured_rows(k, m, present)
            buf = clean.clone()
            keys = inject_counting(torch, buf, checks, 0, length, 8 * c)
            t = min(radius, c // 2)
            a, b, va, vb = blame(torch, do.error_table(k, m, t, present), keys)
            got = check_rebuild(torch, enc, buf, 0, length, k, m, present, radius, a, b, va, vb, keys != 0,
                                [clean[i, :length] for i in lost])
            assert got["damaged_columns"] == length - 1
            assert got["uncorrectable_columns"] == length - 1 - (0 if t == 0 else (k + c) * 255), lost


@pytest.mark.gpu
def test_checked_rebuild_rs_8_6_every_pattern_and_random_syndromes(cuda, swec):
    torch = cuda
    k, m, radius = 8, 6, 2
    present = mask(k + m, RS86_LOST)
    info, checks, _, _, _ = do.punctured_rows(k, m, present)
    table = do.error_table(k, m, radius, present)
    rng = np.random.default_rng(86)
    syn = np.concatenate([table[1], rng.integers(0, 256, (1 << 24, len(checks)), dtype=np.uint8)])
    length = len(syn)
    buf = tiled(torch, k, m, length, seed=86)
    clean_lost = [buf[i, :length].clone() for i in RS86_LOST]
    syn_gpu = torch.from_numpy(syn).to(DEV)
    for i, row in enumerate(checks):
        buf[row, :length] ^= syn_gpu[:, i]
    keys = key_of(torch, syn_gpu)
    a, b, va, vb = blame(torch, table, keys)
    n_table = len(table[0])
    assert (a[:n_table].cpu().numpy() == table[2]).all() and (b[:n_table].cpu().numpy() == table[3]).all()
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    got = check_rebuild(torch, enc, buf, 0, length, k, m, present, radius, a, b, va, vb, keys != 0, clean_lost)
    assert got["damaged_columns"] == length - int((keys == 0).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,lost", [(5, 5, ()), (8, 6, RS86_LOST)])
def test_every_pattern_with_one_syndrome_byte_cleared(cuda, swec, k, m, lost):
    """Every syndrome of the radius-2 table (c = 5 check rows), once with each byte cleared: 14,643,375 columns for
    RS(5,5) (locate and correct), 25,376,325 for RS(8,6) with shard 3 lost (checked rebuild).  These lie next to a
    decodable syndrome, where random damage practically never lands; one with c-2 non-zero bytes, which no pattern
    within radius 2 explains, is uncorrectable however close its bytes come to a data shard's column of P."""
    torch = cuda
    present = mask(k + m, lost) if lost else None
    _, checks, _, _, _ = do.punctured_rows(k, m, present)
    c = len(checks)
    table = do.error_table(k, m, 2, present)
    syn = np.repeat(table[1], c, axis=0)
    syn[np.arange(len(syn)), np.tile(np.arange(c), len(table[1]))] = 0
    length = len(syn)
    buf = tiled(torch, k, m, length, seed=k * 10 + m)
    clean_lost = [buf[i, :length].clone() for i in lost]
    syn_gpu = torch.from_numpy(syn).to(DEV)
    for i, row in enumerate(checks):
        buf[row, :length] ^= syn_gpu[:, i]
    keys = key_of(torch, syn_gpu)
    a, b, va, vb = blame(torch, table, keys)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    if lost:
        got = check_rebuild(torch, enc, buf, 0, length, k, m, present, 2, a, b, va, vb, keys != 0, clean_lost)
    else:
        got = check_locate_and_correct(torch, enc, buf, 0, length, 2, a, b, va, vb, keys != 0)
    weight = (syn_gpu != 0).sum(dim=1)
    assert got["uncorrectable_columns"] >= int(((weight >= 3) & (weight <= c - 2)).sum()) > 0


# ------------------------------------------------------------------------------------------ GPU: the guarantee


def random_damage(n, length, most, rng, ids=None):
    """(errors (length, n) uint8, wrong shards per column): column x has w = 1 + x mod most wrong shards among ids,
    drawn at random, with random non-zero values."""
    ids = np.arange(n) if ids is None else np.asarray(ids)
    w = 1 + np.arange(length) % most
    rank = np.argsort(np.argsort(rng.random((length, len(ids))), axis=1), axis=1)
    hit = np.zeros((length, n), dtype=bool)
    hit[:, ids] = rank < w[:, None]
    err = np.where(hit, rng.integers(1, 256, (length, n)), 0).astype(np.uint8)
    return err, w


def first_two(torch, err):
    """The lowest and second lowest wrong shard of every column (-1: none), on the GPU."""
    hit = torch.from_numpy(err != 0).to(DEV)
    idx = torch.arange(err.shape[1], device=DEV).expand_as(hit)
    big = err.shape[1]
    a = torch.where(hit, idx, big).min(dim=1).values
    b = torch.where(hit & (idx != a[:, None]), idx, big).min(dim=1).values
    return (torch.where(a < big, a, -1).to(torch.int8), torch.where(b < big, b, -1).to(torch.int8))


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 3])
@pytest.mark.parametrize("k,m", SHAPES)
def test_guarantee_against_injected_damage(cuda, swec, k, m, shift):
    torch = cuda
    n, length = k + m, 30_007
    clean = random_set(k, m, length, seed=n * 100 + m)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    for t in radii(m):
        rng = np.random.default_rng(n * 10 + t + shift)
        err, w = random_damage(n, length, m - t, rng)
        buf = buffer(torch, n, length, shift)
        buf[:, shift:shift + length] = torch.from_numpy(np.stack(clean) ^ err.T).to(DEV)
        within = torch.from_numpy(w <= t).to(DEV)
        a, b = first_two(torch, err)
        a, b = torch.where(within, a, -1), torch.where(within, b, -1)
        errs = torch.from_numpy(err).to(DEV)
        rows = torch.arange(length, device=DEV)
        va = torch.where(a >= 0, errs[rows, a.long().clamp(min=0)], 0)
        vb = torch.where(b >= 0, errs[rows, b.long().clamp(min=0)], 0)
        want = check_locate_and_correct(torch, enc, buf, shift, length, t, a, b, va, vb,
                                        torch.ones(length, dtype=torch.bool, device=DEV))
        assert want["uncorrectable_columns"] == int((w > t).sum()) and want["damaged_columns"] == length
        # what correct leaves, stated directly: the clean set where w <= t, the damaged bytes elsewhere
        enc.correct_damage_device(ptrs(buf, shift), length, radius=t, max_ranges=0)
        got = buf[:, shift:shift + length].cpu().numpy()
        assert (got[:, w <= t] == np.stack(clean)[:, w <= t]).all(), t
        assert (got[:, w > t] == (np.stack(clean) ^ err.T)[:, w > t]).all(), t


def patterns_within(torch, n, t, sampled, gen):
    """(a, b, va, vb) of every pattern of 1..t wrong shards: every shard with every value and, at t = 2, every pair of
    shards with every pair of values, or with `sampled` random pairs of values."""
    e = torch.arange(1, 256, device=DEV)
    a = [torch.arange(n, device=DEV).repeat_interleave(255)]
    b = [torch.full((n * 255,), -1, device=DEV)]
    va, vb = [e.repeat(n)], [torch.zeros(n * 255, dtype=torch.int64, device=DEV)]
    if t == 2:
        pairs = torch.combinations(torch.arange(n, device=DEV), 2)
        per = sampled or 255 * 255
        a.append(pairs[:, 0].repeat_interleave(per))
        b.append(pairs[:, 1].repeat_interleave(per))
        if sampled:
            v = torch.randint(1, 256, (2, len(pairs) * per), device=DEV, generator=gen)
            va.append(v[0])
            vb.append(v[1])
        else:
            va.append(e.repeat_interleave(255).repeat(len(pairs)))
            vb.append(e.repeat(255 * len(pairs)))
    return (torch.cat(a).to(torch.int8), torch.cat(b).to(torch.int8), torch.cat(va).to(torch.uint8),
            torch.cat(vb).to(torch.uint8))


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", SHAPES)
def test_every_pattern_within_the_radius(cuda, swec, k, m):
    torch = cuda
    n = k + m
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(n * 31 + m)
    for t in radii(m):
        a, b, va, vb = patterns_within(torch, n, t, 255 if m > 8 else 0, gen)
        length = len(a)
        assert length == n * 255 + (n * (n - 1) // 2 * (255 if m > 8 else 255 * 255) if t == 2 else 0)
        buf = tiled(torch, k, m, length, seed=n + t)
        clean = buf.clone()
        undo_correction(torch, buf, 0, a, b, va, vb, range(n))          # inject: the same XOR
        want = check_locate_and_correct(torch, enc, buf, 0, length, t, a, b, va, vb,
                                        torch.ones(length, dtype=torch.bool, device=DEV))
        assert want["uncorrectable_columns"] == 0 and len(want["shards"]) == n
        enc.correct_damage_device(ptrs(buf, 0), length, radius=t, max_ranges=0)
        assert torch.equal(buf, clean), t
        del buf, clean, a, b, va, vb


def losses(m):
    return sorted({f for f in (1, m - 2, m - 4) if 0 <= f < m})


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", SHAPES)
def test_checked_rebuild_guarantee_against_injected_damage(cuda, swec, k, m):
    torch = cuda
    n, length = k + m, 20_007
    clean = random_set(k, m, length, seed=n * 1000 + m)
    mul = gmul_table(torch)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    for f in losses(m):
        rng = np.random.default_rng(n * 100 + f)
        lost = tuple(sorted(rng.choice(n, size=f, replace=False).tolist()))
        present = mask(n, lost)
        info, checks, _, _, r = do.punctured_rows(k, m, present)
        c = len(checks)
        for radius in (0, 1, 2):
            t = min(radius, c // 2)
            err, w = random_damage(n, length, c - t if t else c, rng, ids=info + checks)
            damaged = np.stack(clean) ^ err.T
            buf = buffer(torch, n, length, 0)
            buf[:, :length] = torch.from_numpy(damaged).to(DEV)
            within = torch.from_numpy(w <= t).to(DEV)
            a, b = first_two(torch, err)
            ida, idb = torch.where(within, a, -1), torch.where(within, b, -1)
            want = without_ok(do.dense_report(ida, idb, torch.ones(length, dtype=torch.bool, device=DEV), n))
            for i in lost:
                buf[i].zero_()
            before = buf.clone()
            got = enc.reconstruct_checked_device(ptrs(buf, 0), present, length, radius=radius, max_ranges=MAX_RANGES)
            assert got == want, (lost, radius)
            assert want["uncorrectable_columns"] == int((w > t).sum())
            for row, i in enumerate(lost):      # the true bytes where w <= t, plain rebuild's elsewhere
                plain = torch.zeros(length, dtype=torch.uint8, device=DEV)
                for j, src in enumerate(info):
                    plain ^= gmul(mul, int(r[row][j]), buf[src, :length])
                true = torch.from_numpy(clean[i]).to(DEV)
                assert torch.equal(buf[i, :length], torch.where(within, true, plain)), (lost, radius, i)
                buf[i].zero_()
            assert torch.equal(buf, before), (lost, radius)


@pytest.mark.gpu
def test_file_level_calls_at_rs_20_12_radius_2(cuda, swec, tmp_path):
    """locate, repair and the checked rebuild with 2 lost (k + c + m = 42 streams a slot) equal the device calls."""
    torch = cuda
    ec = swec.erasure_coding
    k, m, t = 20, 12, 2
    n, length = k + m, 300_007
    clean = random_set(k, m, length, seed=2012)
    rng = np.random.default_rng(2013)
    err, w = random_damage(n, length, 3, rng)
    cols = rng.random(length) < 0.5                  # half the columns damaged, w = 1, 2 or 3
    err[~cols] = 0
    shards = [s ^ e for s, e in zip(clean, err.T)]
    base = str(tmp_path / "v")
    tcr.write_set(base, shards)
    ctx = ec.ECContext(k, m)
    enc = ec.Encoder(k, m, device=0)
    buf = buffer(torch, n, length, 0)
    buf[:, :length] = torch.from_numpy(np.stack(shards)).to(DEV)
    dev = enc.locate_damage_device(ptrs(buf, 0), length, radius=t)
    loc = ec.locate_ec_damage(base, ctx=ctx, radius=t)
    assert without_ok(loc) == dev and not loc["ok"]
    assert dev["damaged_columns"] == int(cols.sum()) and dev["uncorrectable_columns"] == int((cols & (w > t)).sum())
    enc.correct_damage_device(ptrs(buf, 0), length, radius=t)
    assert ec.repair_ec_damage(base, ctx=ctx, radius=t) == loc
    fixed = tcr.file_shards(base, n)
    assert tcr.same(fixed, list(buf[:, :length].cpu().numpy()))
    for sid in range(n):
        assert (fixed[sid][~(cols & (w > t))] == clean[sid][~(cols & (w > t))]).all(), sid
    lost = (5, 27)
    tcr.write_set(base, shards)
    tcr.remove(base, lost)
    buf[:, :length] = torch.from_numpy(np.stack(shards)).to(DEV)
    for i in lost:
        buf[i].zero_()
    present = mask(n, lost)
    dev = enc.reconstruct_checked_device(ptrs(buf, 0), present, length, radius=t)
    rep = ec.rebuild_ec_files_checked(base, ctx=ctx, radius=t)
    assert rep["rebuilt"] == list(lost) and {key: v for key, v in rep.items() if key not in ("rebuilt", "ok")} == dev
    for i in lost:
        assert (np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) == buf[i, :length].cpu().numpy()).all(), i
