"""Repairing damaged EC shards in place: swec_repair_ec_damage (shard files) and swec_correct_damage_device (shards in
HBM), checked against the clean set kept before the damage, and against a correction oracle.  The oracle extends the
exhaustive syndrome table of tests/damage_oracle.py with the error value of every pattern; the kernel and the table both
find the unique pattern within the radius, so they agree byte for byte, miscorrections beyond m - radius included.

cpu: the oracle restores exactly the columns with at most radius wrong shards and leaves t+1 .. m-t unchanged; the
argument rules of both calls; no device; the file checks.  No failure writes a shard file.
gpu: a flipped byte in each of the 14 shards (only the blamed file is written; a second call writes nothing and launches
what locate launches); scattered damage in all 14 shards; overlapping damage at radius 1, then 2; slot boundary, a run
longer than a chunk and the unaligned tail; a shard in an additional directory; O_DIRECT; fuzz at file and device level;
14 x 3 GiB shards in HBM."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import damage_oracle as do  # noqa: E402

from oracle import rs_numpy as rn  # noqa: E402

SEED = 0x2E9A12
GIB = 1 << 30
PAST_NS = 1_000_000_000 * 1_000_000_000    # an mtime no write can produce


def random_set(k, m, length, seed):
    rng = np.random.default_rng(seed)
    data = [rng.integers(0, 256, length, dtype=np.uint8) for _ in range(k)]
    return data + rn.encode(k, m, data)


def damage(shards, columns, n_shards, rng, choose=None):
    """XOR a random non-zero byte into n_shards shards (or the given ones) at every column."""
    for c in columns:
        ids = choose if choose is not None else rng.choice(len(shards), size=n_shards, replace=False)
        for sid in ids:
            shards[int(sid)][c] ^= np.uint8(rng.integers(1, 256))


def write_set(base, shards):
    for i, s in enumerate(shards):
        s.tofile(base + ".ec%02d" % i)


def file_shards(base, n=14):
    return [np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) for i in range(n)]


def same(a, b):
    return len(a) == len(b) and all((x == y).all() for x, y in zip(a, b))


def age(paths):
    """Set every file's mtime far into the past, so that any write shows in st_mtime_ns."""
    for p in paths:
        os.utime(p, ns=(PAST_NS, PAST_NS))


def snapshot(paths):
    return {p: (open(p, "rb").read(), os.stat(p).st_mtime_ns) for p in paths}


def shard_paths(base, n=14):
    return [base + ".ec%02d" % i for i in range(n)]


# ---------------------------------------------------------------------------------------------- correction oracle


@functools.lru_cache(maxsize=None)
def correction_table(k, m, radius):
    """damage_oracle.syndrome_table with the error values: sorted keys, shards a, b (-1: none), values va, vb."""
    h = do.parity_check(k, m)
    n = k + m
    e = np.arange(1, 256, dtype=np.uint8)
    cols = [rn.MUL[e[:, None], h[:, j][None, :]] for j in range(n)]
    keys, a, b, va, vb = [], [], [], [], []
    for j in range(n):
        keys.append(do._keys(cols[j]))
        a.append(np.full(255, j, dtype=np.int8))
        b.append(np.full(255, -1, dtype=np.int8))
        va.append(e)
        vb.append(np.zeros(255, dtype=np.uint8))
    if radius >= 2:
        for x in range(n):
            for y in range(x + 1, n):
                keys.append(do._keys(cols[x][:, None, :] ^ cols[y][None, :, :]).ravel())
                a.append(np.full(255 * 255, x, dtype=np.int8))
                b.append(np.full(255 * 255, y, dtype=np.int8))
                va.append(np.repeat(e, 255))
                vb.append(np.tile(e, 255))
    keys, a, b, va, vb = (np.concatenate(v) for v in (keys, a, b, va, vb))
    order = np.argsort(keys, kind="stable")
    return keys[order], a[order], b[order], va[order], vb[order]


def correct(shards, k, m, radius=1):
    """The shards with every column whose syndrome is in the table corrected; other columns as they were."""
    s = do.syndromes(shards, k, m)
    cols = np.flatnonzero(s.any(axis=1))
    keys, a, b, va, vb = correction_table(k, m, radius)
    q = do._keys(s[cols])
    pos = np.minimum(np.searchsorted(keys, q), len(keys) - 1)
    found = keys[pos] == q
    cols, pos = cols[found], pos[found]
    out = [x.copy() for x in shards]
    for sid in range(k + m):
        for who, val in ((a, va), (b, vb)):
            sel = who[pos] == sid
            out[sid][cols[sel]] ^= val[pos][sel]
    return out


# ------------------------------------------------------------------------------------------ CPU


@pytest.mark.parametrize("k,m", [(10, 4), (6, 3), (12, 4)])
def test_oracle_corrects_within_the_radius_and_leaves_the_rest(k, m):
    rng = np.random.default_rng(k * 10 + m)
    for radius in [r for r in (1, 2) if 2 * r <= m]:
        for wrong in range(1, m - radius + 1):
            clean = random_set(k, m, 3000, seed=wrong)
            shards = [s.copy() for s in clean]
            damage(shards, np.sort(rng.choice(3000, size=200, replace=False)), wrong, rng)
            fixed = correct(shards, k, m, radius)
            if wrong <= radius:
                assert same(fixed, clean), (radius, wrong)
            else:                     # radius < wrong <= m - radius: uncorrectable, left exactly as it was
                assert same(fixed, shards), (radius, wrong)


def test_repair_argument_rules(swec, tmp_path):
    from seaweedfs_b200._native import DamageRange, DamageReport
    ec = swec.erasure_coding
    L = swec.lib()
    base = str(tmp_path / "6")
    shards = random_set(10, 4, 100, 2)
    shards[3][7] ^= 1
    write_set(base, shards)
    age(shard_paths(base))
    before = snapshot(shard_paths(base))
    rep, rng_arr, n, ok = DamageReport(), (DamageRange * 4)(), C.c_int(0), C.c_int(0)
    ptrs = (C.c_void_p * 14)(*([1 << 20] * 14))

    def file_call(k=10, m=4, radius=1, report=C.byref(rep), ranges=rng_arr, cap=4):
        return L.swec_repair_ec_damage(base.encode(), None, 0, k, m, -1, radius, report, ranges, cap, C.byref(n), C.byref(ok))

    def dev_call(enc, radius=1, report=C.byref(rep), ranges=rng_arr, cap=4):
        return L.swec_correct_damage_device(enc._h, ptrs, 4096, radius, report, ranges, cap, C.byref(n), None)

    e104, e63, e101 = ec.Encoder(10, 4, device=-1), ec.Encoder(6, 3, device=-1), ec.Encoder(10, 1, device=-1)
    for call, enc_args in ((file_call, {}), (dev_call, {"enc": e104})):
        for kw in ({"radius": 0}, {"radius": 3}, {"report": None}, {"cap": -1}, {"ranges": None}):
            assert call(**enc_args, **kw) == -1, kw
    assert file_call(k=6, m=3, radius=2) == -1 and b"4 parity shards" in L.swec_last_error()
    assert dev_call(e63, radius=2) == -1
    assert file_call(k=10, m=1) == -1 and dev_call(e101) == -1
    assert dev_call(e63, radius=1) == -7 and dev_call(e104, radius=2) == -7       # valid: on to the device
    assert file_call(radius=2, ranges=None, cap=0) == -7
    assert snapshot(shard_paths(base)) == before


def test_repair_without_a_device(swec, tmp_path):
    ec = swec.erasure_coding
    enc = ec.Encoder(10, 4, device=-1)
    with pytest.raises(swec.SwecError) as e:
        enc.correct_damage_device([1 << 20] * 14, 4096)
    assert e.value.name == "SWEC_ERR_NO_DEVICE"
    base = str(tmp_path / "5")
    shards = random_set(10, 4, 5000, 1)
    shards[12][4000] ^= 0x10
    write_set(base, shards)
    age(shard_paths(base))
    before = snapshot(shard_paths(base))
    with pytest.raises(swec.SwecError) as e:
        ec.repair_ec_damage(base, device=-1)          # the files check out; the device work cannot start
    assert e.value.name == "SWEC_ERR_NO_DEVICE"
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(swec.SwecError) as e:
            ec.repair_ec_damage(base, device=0)
        assert e.value.name == "SWEC_ERR_NO_DEVICE"
    assert snapshot(shard_paths(base)) == before


def test_repair_file_checks(swec, tmp_path):
    """Both checks come before any device work (device=-1 would fail there) and before anything is written."""
    ec = swec.erasure_coding
    device = -1
    base = str(tmp_path / "8")
    shards = random_set(10, 4, 1000, 3)
    shards[2][10] ^= 0xFF
    write_set(base, shards)
    with open(base + ".ec11", "ab") as f:
        f.write(b"x")
    age(shard_paths(base))
    before = snapshot(shard_paths(base))
    with pytest.raises(swec.SwecError) as e:
        ec.repair_ec_damage(base, device=device)
    assert e.value.name == "SWEC_ERR_SHARD_SIZE" and "expected 1000 actual 1001" in str(e.value)
    assert snapshot(shard_paths(base)) == before
    os.remove(base + ".ec07")
    paths = [p for p in shard_paths(base) if os.path.exists(p)]
    before = snapshot(paths)
    with pytest.raises(swec.SwecError) as e:
        ec.repair_ec_damage(base, device=device)
    assert e.value.name == "SWEC_ERR_TOO_FEW_SHARDS" and ".ec07" in str(e.value)
    assert snapshot(paths) == before


# ------------------------------------------------------------------------------------------ GPU


def flip(path, off, mask=0x40):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ mask]))


def without_ok(rep):
    return {key: v for key, v in rep.items() if key != "ok"}


def mtimes(paths):
    return [os.stat(p).st_mtime_ns for p in paths]


@pytest.mark.gpu
def test_one_flipped_byte_per_shard(cuda, swec, oracle, tmp_path):
    ec = swec.erasure_coding
    L = swec.lib()
    size = 12_345_678
    base = str(tmp_path / "21")
    oracle.synth(0, size, SEED).tofile(base + ".dat")
    ec.write_ec_files(base)
    clean = file_shards(base)
    shard_len = len(clean[0])
    paths = shard_paths(base)
    for sid in range(14):
        off = (777_777 * (sid + 1)) % shard_len
        flip(paths[sid], off)
        age(paths)
        rep = ec.repair_ec_damage(base)
        assert rep["ok"] and rep["damaged_columns"] == 1 and rep["uncorrectable_columns"] == 0
        assert rep["shards"] == {sid: (1, off, off)}
        assert rep["ranges"] == [(sid, off // 4096 * 4096, min(4096, shard_len - off // 4096 * 4096))]
        assert same(file_shards(base), clean), sid
        assert [t != PAST_NS for t in mtimes(paths)] == [i == sid for i in range(14)], sid
    # a repaired set: nothing to do, nothing written, the launches of a locate call
    age(paths)
    n0 = L.swec_kernel_launches()
    rep = ec.repair_ec_damage(base)
    n1 = L.swec_kernel_launches()
    loc = ec.locate_ec_damage(base)
    n2 = L.swec_kernel_launches()
    assert rep == loc and rep["ok"] and rep["damaged_columns"] == 0
    assert n1 - n0 == n2 - n1 > 0
    assert mtimes(paths) == [PAST_NS] * 14


@pytest.mark.gpu
def test_scattered_damage_in_all_14_shards(cuda, swec, oracle, tmp_path):
    """Every shard damaged at its own pages: 14 shards blamed, more than the 4 a rebuild can replace."""
    ec = swec.erasure_coding
    size = 31_000_000
    base = str(tmp_path / "s")
    dat = oracle.synth(0, size, SEED + 1)
    dat.tofile(base + ".dat")
    ec.write_ec_files(base)
    clean = file_shards(base)
    shard_len = len(clean[0])
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(5)
    for sid in range(14):
        for page in (3 * sid, 3 * sid + 1, 50 + 17 * sid):     # disjoint runs, no two shards share a page
            cols = np.sort(rng.choice(4096, size=300, replace=False)) + page * 4096
            damage(shards, cols[cols < shard_len], 1, rng, choose=[sid])
    write_set(base, shards)
    want = do.locate(shards, 10, 4)
    assert len(want["shards"]) == 14 and want["uncorrectable_columns"] == 0
    rep = ec.repair_ec_damage(base)
    assert rep == {**want, "ok": True}
    assert same(file_shards(base), clean)
    assert ec.verify_ec_files(base) == (True, [0, 0, 0, 0])
    out = str(tmp_path / "back")
    ec.write_dat_file(out, size, shard_paths(base, 10))
    assert (np.fromfile(out + ".dat", dtype=np.uint8) == dat).all()


@pytest.mark.gpu
def test_overlapping_damage_radius_1_then_2(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    length = 300_000
    clean = random_set(10, 4, length, 21)
    rng = np.random.default_rng(22)
    shards = [s.copy() for s in clean]
    damage(shards, np.arange(10_000, 60_000), 1, rng, choose=[2])
    damage(shards, np.arange(40_000, 90_000), 1, rng, choose=[12])      # overlap 40,000..59,999
    base = str(tmp_path / "4")
    write_set(base, shards)
    r1 = ec.repair_ec_damage(base, radius=1)
    assert r1 == {**do.locate(shards, 10, 4, 1), "ok": False}
    assert r1["shards"] == {2: (30_000, 10_000, 39_999), 12: (30_000, 60_000, 89_999)}
    after1 = file_shards(base)
    assert same(after1, correct(shards, 10, 4, 1))
    for sid in range(14):                                               # the overlap is left as it was
        assert (after1[sid][40_000:60_000] == shards[sid][40_000:60_000]).all()
        assert (after1[sid][:40_000] == clean[sid][:40_000]).all() and (after1[sid][60_000:] == clean[sid][60_000:]).all()
    r2 = ec.repair_ec_damage(base, radius=2)
    assert r2 == {**do.locate(after1, 10, 4, 2), "ok": True}
    assert r2["shards"] == {2: (20_000, 40_000, 59_999), 12: (20_000, 40_000, 59_999)}
    assert same(file_shards(base), clean)


@pytest.mark.gpu
def test_slot_boundary_long_run_and_tail(cuda, swec, tmp_path, monkeypatch):
    ec = swec.erasure_coding
    monkeypatch.setenv("SWEC_FILE_CHUNK", str(64 << 10))
    length = 1_000_003                       # not a multiple of 16: the last columns take the byte path
    clean = random_set(10, 4, length, 11)
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(12)
    first = 3 * (64 << 10) - 2000            # 4 KiB + 77 bytes straddling the boundary of the third slot
    damage(shards, np.arange(first, first + 4096 + 77), 1, rng, choose=[3])
    damage(shards, np.arange(400_000, 400_000 + 150_000), 1, rng, choose=[11])   # longer than two chunks
    damage(shards, np.arange(length - 1000, length), 1, rng, choose=[3])        # ends on the last byte
    damage(shards, [length - 1], 1, rng, choose=[13])                            # same column, another shard
    base = str(tmp_path / "3")
    write_set(base, shards)
    want = do.locate(shards, 10, 4)
    rep = ec.repair_ec_damage(base)
    assert rep == {**want, "ok": want["uncorrectable_columns"] == 0}
    assert rep["uncorrectable_columns"] == 1 and rep["first_uncorrectable"] == length - 1
    fixed = file_shards(base)
    assert same(fixed, correct(shards, 10, 4))
    for sid in range(14):
        assert (fixed[sid][:-1] == clean[sid][:-1]).all(), sid
        assert fixed[sid][-1] == shards[sid][-1], sid          # the uncorrectable column, as it was
    rep2 = ec.repair_ec_damage(base, radius=2)
    assert rep2["ok"] and rep2["shards"] == {3: (1, length - 1, length - 1), 13: (1, length - 1, length - 1)}
    assert same(file_shards(base), clean)


@pytest.mark.gpu
def test_shard_in_an_additional_directory(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    length = 500_000
    clean = random_set(10, 4, length, 41)
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(42)
    damage(shards, np.arange(70_000, 80_000), 1, rng, choose=[9])
    damage(shards, np.arange(200, 300), 1, rng, choose=[1])
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    base, other = str(tmp_path / "a" / "7"), str(tmp_path / "b" / "7")
    for i, s in enumerate(shards):                              # shards 8..13 live in the other directory
        s.tofile((other if i >= 8 else base) + ".ec%02d" % i)
    rep = ec.repair_ec_damage(base, additional_dirs=[str(tmp_path / "b")])
    assert rep["ok"] and set(rep["shards"]) == {1, 9}
    assert not os.path.exists(base + ".ec09")                   # repaired where it was found
    got = [np.fromfile((other if i >= 8 else base) + ".ec%02d" % i, dtype=np.uint8) for i in range(14)]
    assert same(got, clean)


@pytest.mark.gpu
def test_repair_with_o_direct(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    L = swec.lib()
    length = 3 * (8 << 20) + 4096 * 5 + 123
    clean = random_set(10, 4, length, 51)
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(52)
    damage(shards, np.arange(8 << 20, (8 << 20) + 3 * 4096), 1, rng, choose=[0])   # whole pages at a slot start
    damage(shards, np.arange(100_000, 100_050), 1, rng, choose=[10])
    damage(shards, np.arange(length - 200, length), 1, rng, choose=[6])             # the clipped last page
    base = str(tmp_path / "d")
    write_set(base, shards)
    assert L.swec_set_option(b"file_direct_io", 3) == 0
    try:
        rep = ec.repair_ec_damage(base)
    finally:
        assert L.swec_set_option(b"file_direct_io", int(os.environ.get("SWEC_FILE_DIRECT", "0")) & 3) == 0
    assert rep == {**do.locate(shards, 10, 4), "ok": True}
    assert same(file_shards(base), clean)


def fuzz_set(k, m, length, seed):
    rng = np.random.default_rng(seed)
    shards = random_set(k, m, length, seed)
    cols = np.sort(rng.choice(length, size=length // 3, replace=False))
    for c in cols:
        damage(shards, [c], int(rng.integers(1, 4)), rng)
    return shards


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,radii", [(10, 4, (1, 2)), (6, 3, (1,))])
def test_fuzz_against_the_correction_oracle(cuda, swec, tmp_path, k, m, radii):
    """Random XOR damage of 1-3 shards per column, file level and device level (aligned and unaligned pointers)."""
    ec = swec.erasure_coding
    torch = cuda
    length = 6_000 + 7
    shards = fuzz_set(k, m, length, seed=k + m + 100)
    enc = ec.Encoder(k, m, device=0)
    for radius in radii:
        want = do.locate(shards, k, m, radius)
        fixed = correct(shards, k, m, radius)
        assert want["damaged_columns"] == length // 3
        base = str(tmp_path / ("f%d" % radius))
        write_set(base, shards)
        rep = ec.repair_ec_damage(base, ctx=ec.ECContext(k, m), radius=radius)
        assert rep == {**want, "ok": want["uncorrectable_columns"] == 0}
        assert same(file_shards(base, k + m), fixed), radius
        for shift in (0, 1, 5):
            bufs = [torch.zeros(length + 16, dtype=torch.uint8, device="cuda") for _ in shards]
            for b, s in zip(bufs, shards):
                b[shift:shift + length] = torch.from_numpy(s).cuda()
            got = enc.correct_damage_device([b.data_ptr() + shift for b in bufs], length, radius=radius)
            assert got == without_ok(want), (radius, shift)
            back = [b[shift:shift + length].cpu().numpy() for b in bufs]
            assert same(back, fixed), (radius, shift)
            assert all((b[:shift] == 0).all() and (b[shift + length:] == 0).all() for b in bufs), (radius, shift)


@pytest.mark.gpu
def test_full_size_shards_in_hbm(cuda, swec):
    """14 x 3 GiB shards (a 30 GiB volume's) in HBM, damaged at the sites of the locate test, corrected in place."""
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

    def digests():
        out = []
        for s in shards:
            d = C.c_uint64(0)
            swec._native.check(L.swec_digest_device(0, s.data_ptr(), n, C.byref(d), None))
            out.append(d.value)
        return out

    before = digests()
    ptrs = [s.data_ptr() for s in shards]
    rep = enc.correct_damage_device(ptrs, n)
    assert rep["damaged_columns"] == 0 and rep["shards"] == {} and digests() == before
    run = 1_500_000_000
    for radius in (1, 2):
        shards[12][run:run + (1 << 20)] ^= 0x11        # 1 MiB run in parity shard 12, not page aligned
        shards[7][n - 1] ^= 0x80                        # the last byte of a data shard
        shards[0][5] ^= 1
        shards[13][2 * GIB] ^= 0xFF
        torch.cuda.synchronize()
        assert digests() != before
        rep = enc.correct_damage_device(ptrs, n, radius=radius)
        assert rep["damaged_columns"] == (1 << 20) + 3 and rep["uncorrectable_columns"] == 0
        assert rep["shards"] == {0: (1, 5, 5), 7: (1, n - 1, n - 1), 12: (1 << 20, run, run + (1 << 20) - 1),
                                 13: (1, 2 * GIB, 2 * GIB)}
        assert digests() == before, radius
        assert enc.locate_damage_device(ptrs, n)["damaged_columns"] == 0
    del shards
    torch.cuda.empty_cache()
