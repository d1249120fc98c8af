"""Locating the wrong shard when EC parity does not match: swec_locate_ec_damage (shard files) and
swec_locate_damage_device (shards in HBM), checked against tests/damage_oracle.py (exhaustive search over every single
shard and pair of shards with every error value).

cpu: the oracle recovers injected damage and calls t+1 .. m-t wrong shards uncorrectable; the MDS property the guarantee
rests on; struct layout against the header; argument and file checks; no device.
gpu: clean set; a flipped byte in each of the 14 shards; runs across a pipeline slot boundary and in the tail; overlapping
damage at radius 1 and 2; fuzz at file and device level (unaligned pointers, RS(6,3)); the range cap; delete-and-rebuild
round trip; 14 x 3 GiB shards in HBM."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import damage_oracle as do  # noqa: E402

from oracle import rs_numpy as rn  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 0xDA3A6E
GIB = 1 << 30


def random_set(k, m, length, seed):
    rng = np.random.default_rng(seed)
    data = [rng.integers(0, 256, length, dtype=np.uint8) for _ in range(k)]
    return data + rn.encode(k, m, data)


def damage(shards, columns, n_shards, rng, choose=None):
    """XOR a random non-zero byte into n_shards shards (or the given ones) at every column; returns the shards hit."""
    hit = []
    for c in columns:
        ids = choose if choose is not None else rng.choice(len(shards), size=n_shards, replace=False)
        for sid in ids:
            shards[int(sid)][c] ^= np.uint8(rng.integers(1, 256))
        hit.append(sorted(int(s) for s in ids))
    return hit


def write_set(base, shards):
    for i, s in enumerate(shards):
        s.tofile(base + ".ec%02d" % i)


# ------------------------------------------------------------------------------------------ CPU


@pytest.mark.parametrize("k,m", [(10, 4), (6, 3), (12, 4)])
def test_oracle_recovers_what_was_injected(k, m):
    rng = np.random.default_rng(k * 100 + m)
    for radius in [r for r in (1, 2) if 2 * r <= m]:
        for wrong in range(1, m - radius + 1):
            shards = random_set(k, m, 3000, seed=wrong)
            cols = np.sort(rng.choice(3000, size=200, replace=False))
            hit = damage(shards, cols, wrong, rng)
            got_cols, a, b = do.locate_columns(shards, k, m, radius)
            assert (got_cols == cols).all()
            if wrong <= radius:          # located exactly
                for want, x, y in zip(hit, a, b):
                    assert sorted(int(v) for v in (x, y) if v >= 0) == want
            else:                        # radius < wrong <= m - radius: uncorrectable, nobody blamed
                assert (a < 0).all() and (b < 0).all()
            rep = do.locate(shards, k, m, radius)
            assert rep["damaged_columns"] == 200 and not rep["ok"]


@pytest.mark.parametrize("k,m", [(10, 4), (6, 3), (12, 4), (3, 2)])
def test_parity_check_columns_are_independent(k, m):
    """The guarantee rests on the code being MDS: any m columns of [P | I] are independent."""
    import itertools
    h = do.parity_check(k, m)
    for cols in itertools.combinations(range(k + m), 2):
        assert do.gf_rank(h[:, cols]) == 2, cols
    if m >= 4:
        for cols in itertools.combinations(range(k + m), 4):
            assert do.gf_rank(h[:, cols]) == 4, cols


def test_damage_structs_match_the_header(swec, tmp_path):
    from seaweedfs_b200._native import DamageRange, DamageReport
    src = tmp_path / "s.c"
    fields = [("swec_damage_report", f) for f in ("damaged_columns", "first_uncorrectable", "last_uncorrectable",
                                                  "shard_bytes", "shard_first", "shard_last")]
    fields += [("swec_damage_range", f) for f in ("reserved", "offset", "length")]
    body = ", ".join(f"offsetof({t}, {f})" for t, f in fields)
    fmt = " ".join(["%zu"] * (len(fields) + 2))
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "swec.h"\n'
                   f'int main(void){{printf("{fmt}\\n", sizeof(swec_damage_report), sizeof(swec_damage_range), {body});'
                   'return 0;}\n')
    exe = str(tmp_path / "s")
    subprocess.run(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", exe, str(src)], check=True)
    got = [int(x) for x in subprocess.run([exe], check=True, stdout=subprocess.PIPE, text=True).stdout.split()]
    want = [C.sizeof(DamageReport), C.sizeof(DamageRange)]
    want += [getattr(DamageReport if t == "swec_damage_report" else DamageRange, f).offset for t, f in fields]
    assert got == want


def test_locate_without_a_device(swec, tmp_path):
    ec = swec.erasure_coding
    enc = ec.Encoder(10, 4, device=-1)
    with pytest.raises(swec.SwecError) as e:
        enc.locate_damage_device([1 << 20] * 14, 4096)
    assert e.value.name == "SWEC_ERR_NO_DEVICE"
    base = str(tmp_path / "5")
    write_set(base, random_set(10, 4, 5000, 1))
    with pytest.raises(swec.SwecError) as e:
        ec.locate_ec_damage(base, device=-1)          # the files check out; the device work cannot start
    assert e.value.name == "SWEC_ERR_NO_DEVICE"
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(swec.SwecError) as e:
            ec.locate_ec_damage(base, device=0)
        assert e.value.name == "SWEC_ERR_NO_DEVICE"


def test_locate_argument_rules(swec, tmp_path):
    from seaweedfs_b200._native import DamageRange, DamageReport
    ec = swec.erasure_coding
    L = swec.lib()
    base = str(tmp_path / "6")
    write_set(base, random_set(10, 4, 100, 2))
    rep, rng_arr, n, ok = DamageReport(), (DamageRange * 4)(), C.c_int(0), C.c_int(0)
    ptrs = (C.c_void_p * 14)(*([1 << 20] * 14))

    def file_call(k=10, m=4, radius=1, report=C.byref(rep), ranges=rng_arr, cap=4):
        return L.swec_locate_ec_damage(base.encode(), None, 0, k, m, -1, radius, report, ranges, cap, C.byref(n), C.byref(ok))

    def dev_call(enc, radius=1, report=C.byref(rep), ranges=rng_arr, cap=4):
        return L.swec_locate_damage_device(enc._h, ptrs, 4096, radius, report, ranges, cap, C.byref(n), None)

    e104, e63, e101 = ec.Encoder(10, 4, device=-1), ec.Encoder(6, 3, device=-1), ec.Encoder(10, 1, device=-1)
    for call, enc_args in ((file_call, {}), (dev_call, {"enc": e104})):
        for kw in ({"radius": 0}, {"radius": 3}, {"report": None}, {"cap": -1}, {"ranges": None}):
            assert call(**enc_args, **kw) == -1, kw
    assert file_call(k=6, m=3, radius=2) == -1 and b"4 parity shards" in L.swec_last_error()
    assert dev_call(e63, radius=2) == -1
    assert file_call(k=10, m=1) == -1 and dev_call(e101) == -1
    assert dev_call(e63, radius=1) == -7 and dev_call(e104, radius=2) == -7       # valid: on to the device
    assert file_call(radius=2, ranges=None, cap=0) == -7


def test_locate_file_checks(swec, tmp_path):
    ec = swec.erasure_coding
    base = str(tmp_path / "8")
    write_set(base, random_set(10, 4, 1000, 3))
    with open(base + ".ec11", "ab") as f:
        f.write(b"x")
    with pytest.raises(swec.SwecError) as e:
        ec.locate_ec_damage(base, device=-1)
    assert e.value.name == "SWEC_ERR_SHARD_SIZE" and "expected 1000 actual 1001" in str(e.value)
    os.remove(base + ".ec07")
    with pytest.raises(swec.SwecError) as e:
        ec.locate_ec_damage(base, device=-1)
    assert e.value.name == "SWEC_ERR_TOO_FEW_SHARDS" and ".ec07" in str(e.value)


# ------------------------------------------------------------------------------------------ GPU


def flip(path, off, mask=0x40):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ mask]))


def file_shards(base, n=14):
    return [np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) for i in range(n)]


def without_ok(rep):
    return {key: v for key, v in rep.items() if key != "ok"}


@pytest.mark.gpu
def test_clean_set_and_one_flipped_byte_per_shard(cuda, swec, oracle, tmp_path):
    ec = swec.erasure_coding
    size = 12_345_678
    base = str(tmp_path / "21")
    oracle.synth(0, size, SEED).tofile(base + ".dat")
    ec.write_ec_files(base)
    shard_len = os.path.getsize(base + ".ec00")
    rep = ec.locate_ec_damage(base)
    assert rep["ok"] and rep["columns"] == shard_len and rep["damaged_columns"] == 0
    assert rep["shards"] == {} and rep["ranges"] == [] and rep["n_ranges"] == 0
    assert rep["uncorrectable_columns"] == 0 and rep["first_uncorrectable"] == rep["last_uncorrectable"] == -1
    for sid in range(14):
        off = (777_777 * (sid + 1)) % shard_len
        flip(base + ".ec%02d" % sid, off)
        rep = ec.locate_ec_damage(base)
        assert not rep["ok"] and rep["damaged_columns"] == 1 and rep["uncorrectable_columns"] == 0
        assert rep["shards"] == {sid: (1, off, off)}
        assert rep["ranges"] == [(sid, off // 4096 * 4096, min(4096, shard_len - off // 4096 * 4096))]
        if sid == 3:
            assert ec.verify_ec_files(base) == (False, [1, 1, 1, 1])   # verify alone names every parity shard
        flip(base + ".ec%02d" % sid, off)
    assert ec.locate_ec_damage(base)["ok"]


@pytest.mark.gpu
def test_runs_across_a_slot_boundary_and_in_the_tail(cuda, swec, tmp_path, monkeypatch):
    ec = swec.erasure_coding
    monkeypatch.setenv("SWEC_FILE_CHUNK", str(64 << 10))
    length = 1_000_003                       # not a multiple of 16: the last 3 columns take the byte path
    shards = random_set(10, 4, length, 11)
    base = str(tmp_path / "3")
    rng = np.random.default_rng(12)
    first = 3 * (64 << 10) - 2000            # 4 KiB + 77 bytes straddling the boundary of the third slot
    run1 = np.arange(first, first + 4096 + 77)
    run2 = np.arange(length - 1000, length)  # ends on the shard's last byte
    damage(shards, run1, 1, rng, choose=[3])
    damage(shards, run2, 1, rng, choose=[3])
    write_set(base, shards)
    rep = ec.locate_ec_damage(base)
    assert rep == do.locate(shards, 10, 4)
    assert rep["shards"] == {3: (len(run1) + len(run2), first, length - 1)}
    p0 = first // 4096 * 4096
    assert rep["ranges"] == [(3, p0, (run1[-1] // 4096 + 1) * 4096 - p0),
                             (3, run2[0] // 4096 * 4096, length - run2[0] // 4096 * 4096)]


@pytest.mark.gpu
def test_overlapping_damage_in_two_and_three_shards(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    length = 300_000
    clean = random_set(10, 4, length, 21)
    rng = np.random.default_rng(22)
    shards = [s.copy() for s in clean]
    damage(shards, np.arange(10_000, 60_000), 1, rng, choose=[2])
    damage(shards, np.arange(40_000, 90_000), 1, rng, choose=[12])      # overlap 40,000..59,999
    base = str(tmp_path / "4")
    write_set(base, shards)
    r1 = ec.locate_ec_damage(base, radius=1)
    assert r1 == do.locate(shards, 10, 4, 1)
    assert r1["shards"] == {2: (30_000, 10_000, 39_999), 12: (30_000, 60_000, 89_999)}
    assert (r1["uncorrectable_columns"], r1["first_uncorrectable"], r1["last_uncorrectable"]) == (20_000, 40_000, 59_999)
    r2 = ec.locate_ec_damage(base, radius=2)
    assert r2 == do.locate(shards, 10, 4, 2)
    assert r2["shards"] == {2: (50_000, 10_000, 59_999), 12: (50_000, 40_000, 89_999)}
    assert r2["uncorrectable_columns"] == 0 and r2["damaged_columns"] == 80_000
    # a third shard over part of the overlap: radius 1 calls it uncorrectable and blames nobody there
    damage(shards, np.arange(50_000, 55_000), 1, rng, choose=[7])
    write_set(base, shards)
    r3 = ec.locate_ec_damage(base, radius=1)
    assert r3 == do.locate(shards, 10, 4, 1)
    assert r3["shards"] == {2: (30_000, 10_000, 39_999), 12: (30_000, 60_000, 89_999)}
    assert r3["uncorrectable_columns"] == 20_000


def fuzz_set(k, m, length, seed):
    rng = np.random.default_rng(seed)
    shards = random_set(k, m, length, seed)
    cols = np.sort(rng.choice(length, size=length // 3, replace=False))
    for c in cols:
        damage(shards, [c], int(rng.integers(1, 4)), rng)
    return shards


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,radii", [(10, 4, (1, 2)), (6, 3, (1,))])
def test_fuzz_against_the_oracle(cuda, swec, tmp_path, k, m, radii):
    """Random XOR damage of 1-3 shards per column, file level and device level (aligned and unaligned pointers).
    Both sides search the same radius, so they agree exactly, misattribution beyond m - radius included."""
    ec = swec.erasure_coding
    torch = cuda
    length = 6_000 + 7
    shards = fuzz_set(k, m, length, seed=k + m)
    base = str(tmp_path / "f")
    write_set(base, shards)
    enc = ec.Encoder(k, m, device=0)
    for radius in radii:
        want = do.locate(shards, k, m, radius)
        assert want["damaged_columns"] == length // 3
        assert ec.locate_ec_damage(base, ctx=ec.ECContext(k, m), radius=radius) == want
        for shift in (0, 1, 5):
            bufs = [torch.zeros(length + 16, dtype=torch.uint8, device="cuda") for _ in shards]
            for b, s in zip(bufs, shards):
                b[shift:shift + length] = torch.from_numpy(s).cuda()
            got = enc.locate_damage_device([b.data_ptr() + shift for b in bufs], length, radius=radius)
            assert got == without_ok(want), (radius, shift)


@pytest.mark.gpu
def test_ranges_cap_keeps_the_total(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    length = 200 * 4096
    shards = random_set(10, 4, length, 31)
    rng = np.random.default_rng(32)
    damage(shards, np.arange(0, length, 2 * 4096), 1, rng, choose=[5])   # 100 separate pages
    base = str(tmp_path / "c")
    write_set(base, shards)
    full = ec.locate_ec_damage(base)
    assert full["n_ranges"] == 100 and len(full["ranges"]) == 100
    few = ec.locate_ec_damage(base, max_ranges=7)
    assert few["n_ranges"] == 100 and few["ranges"] == full["ranges"][:7]
    none = ec.locate_ec_damage(base, max_ranges=0)
    assert none["n_ranges"] == 100 and none["ranges"] == []


@pytest.mark.gpu
def test_remedy_delete_the_blamed_shard_and_rebuild(cuda, swec, oracle, tmp_path):
    ec = swec.erasure_coding
    size = 5_000_000
    base = str(tmp_path / "r")
    oracle.synth(0, size, SEED + 1).tofile(base + ".dat")
    ec.write_ec_files(base)
    clean = file_shards(base)
    for sid, off in ((3, 123_457), (3, 200_000), (11, 9)):
        flip(base + ".ec%02d" % sid, off, 0x5A)
    rep = ec.locate_ec_damage(base)
    assert set(rep["shards"]) == {3, 11} and rep["uncorrectable_columns"] == 0
    for sid in rep["shards"]:
        os.remove(base + ".ec%02d" % sid)
    assert ec.rebuild_ec_files(base) == [3, 11]
    assert ec.verify_ec_files(base) == (True, [0, 0, 0, 0])
    assert ec.locate_ec_damage(base)["ok"]
    for a, b in zip(file_shards(base), clean):
        assert (a == b).all()


@pytest.mark.gpu
def test_full_size_shards_in_hbm(cuda, swec):
    """14 x 3 GiB shards (a 30 GiB volume's) in HBM: a clean pass, then a few damaged sites located exactly."""
    torch = cuda
    ec = swec.erasure_coding
    L = swec.lib()
    n = 3 * GIB
    torch.cuda.empty_cache()
    shards = [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(14)]
    for i in range(10):
        swec._native.check(L.swec_synth_fill_device(0, shards[i].data_ptr(), i * n, n, SEED, None))
    enc = ec.Encoder(10, 4, device=0)
    enc.encode_device([s.data_ptr() for s in shards[:10]], [s.data_ptr() for s in shards[10:]], n)
    enc.synchronize()
    ptrs = [s.data_ptr() for s in shards]
    rep = enc.locate_damage_device(ptrs, n)
    assert rep["damaged_columns"] == 0 and rep["shards"] == {} and rep["ranges"] == []
    run = 1_500_000_000
    shards[12][run:run + (1 << 20)] ^= 0x11        # 1 MiB run in parity shard 12, not page aligned
    shards[7][n - 1] ^= 0x80                        # the last byte of a data shard
    shards[0][5] ^= 1
    shards[13][2 * GIB] ^= 0xFF
    torch.cuda.synchronize()
    for radius in (1, 2):
        rep = enc.locate_damage_device(ptrs, n, radius=radius)
        assert rep["damaged_columns"] == (1 << 20) + 3 and rep["uncorrectable_columns"] == 0
        assert rep["shards"] == {0: (1, 5, 5), 7: (1, n - 1, n - 1), 12: (1 << 20, run, run + (1 << 20) - 1),
                                 13: (1, 2 * GIB, 2 * GIB)}
        p0 = run // 4096 * 4096
        assert rep["ranges"] == [(0, 0, 4096), (7, n - 4096, 4096),
                                 (12, p0, ((run + (1 << 20) - 1) // 4096 + 1) * 4096 - p0), (13, 2 * GIB, 4096)]
    del shards
    torch.cuda.empty_cache()
