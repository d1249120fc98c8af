"""Which needles located EC damage hits: swec_locate_needle_damage_device and swec_ec_volume_locate_needle_damage.

Expected values come from the existing oracles and share nothing with the method:
- damage_oracle.decode_columns gives the blame and the uncorrectable columns of every damaged column;
- a plain Python walk of encodeDatFile's striping (blocks in the order the encoder lays them down), or the oracle's
  LocateData intervals for a mounted volume, maps each data-shard byte to its .dat offset;
- needle_oracle.actual_size sizes the records, and the owner of a byte is found with bisect.
Every field of every record, unowned, the report and the ranges are compared, and both invariants are asserted.

cpu: the inverse striping of stripe_map.h, compiled for the host, against the oracle's forward striping (every byte of
every data shard over a grid of geometries) and against LocateData; argument rules and their order; file checks of the
handle call; the kernel ledger of needle_damage.cu; the pinned SASS of the locate kernel.
"""
from __future__ import annotations

import bisect
import ctypes as C
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import damage_oracle as do  # noqa: E402
import needle_oracle as no  # noqa: E402

from oracle import rs_numpy as rn  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_IDX = os.path.join(ROOT, "tests", "golden", "fixtures", "1.idx")
REF_DAT = os.path.join(ROOT, "oracle", "_ref", "1.dat")
MIB, GIB = 1 << 20, 1 << 30
PIECE = 256 * MIB
SEED = 0x4EED1E


# ---------------------------------------------------------------------------------------------- oracle side


def walk_blocks(k, dat_size, large, small):
    """(shard, shard offset, .dat offset, bytes) of every block in the order encodeDatFile lays them down: rows of k
    large blocks while a whole large row remains, then rows of k small blocks, the last one cut at the end of the .dat."""
    out, d, x = [], 0, 0
    while dat_size - d >= large * k:
        out += [(i, x, d + i * large, large) for i in range(k)]
        d, x = d + large * k, x + large
    while d < dat_size:
        out += [(i, x, d + i * small, max(0, min(small, dat_size - d - i * small))) for i in range(k)]
        d, x = d + small * k, x + small
    return out


class Striping:
    """.dat offset of byte x of data shard i, from walk_blocks (-1: padding)."""

    def __init__(self, k, dat_size, large, small):
        self.per = [[] for _ in range(k)]
        for i, x, d, n in walk_blocks(k, dat_size, large, small):
            self.per[i].append((x, d, n))
        self.starts = [[b[0] for b in p] for p in self.per]

    def __call__(self, i, x):
        j = bisect.bisect_right(self.starts[i], x) - 1
        if j < 0:
            return -1
        bx, d, n = self.per[i][j]
        return d + (x - bx) if x - bx < n else -1

    def shard_pos(self, d):
        for i, p in enumerate(self.per):
            for bx, bd, n in p:
                if bd <= d < bd + n:
                    return i, bx + d - bd
        raise ValueError(d)


class Owners:
    """The live record owning a .dat offset: the one with the greatest offset not above it (the later entry on a tie),
    when the offset lies inside it."""

    def __init__(self, records, version=3):
        order = sorted(range(len(records)), key=lambda j: records[j][1])
        self.order = order
        self.offs = [records[j][1] for j in order]
        self.ends = [records[j][1] + (no.actual_size(records[j][2], version) if records[j][2] >= 0 else 0) for j in order]

    def __call__(self, d):
        if d < 0:
            return -1
        p = bisect.bisect_right(self.offs, d) - 1
        return self.order[p] if p >= 0 and d < self.ends[p] else -1


def expected(shards, k, m, radius, records, dat_offset):
    """(report, per-record [mask, damaged, uncorrectable], unowned) for shards as found."""
    cols, a, b, _, _, _ = do.decode_columns(shards, k, m, radius)
    rep = do.report(len(shards[0]), k + m, cols, a, b)
    owner = Owners(records)
    per = [[0, 0, 0] for _ in records]
    unowned = [0, 0]
    for c, x, y in zip(cols.tolist(), a.tolist(), b.tolist()):
        unc = x < 0 and y < 0
        hit = range(k) if unc else [s for s in (x, y) if 0 <= s < k]
        for i in hit:
            j = owner(dat_offset(i, c))
            if j < 0:
                unowned[int(unc)] += 1
            else:
                per[j][0] |= 1 << i
                per[j][2 if unc else 1] += 1
    return rep, per, unowned


def check_invariants(res, k, records_out):
    assert sum(r["damaged_bytes"] for r in records_out) + res["unowned"][0] == \
        sum(v[0] for s, v in res["shards"].items() if s < k)
    assert sum(r["uncorrectable_bytes"] for r in records_out) + res["unowned"][1] == k * res["uncorrectable_columns"]


def compare(res, want, records_in, k, all_records=True):
    rep, per, unowned = want
    got = {key: res[key] for key in rep if key != "ok"}
    assert got == {key: v for key, v in rep.items() if key != "ok"}
    assert res["unowned"] == unowned
    if all_records:
        assert [(r["needle_id"], r["offset"], r["size"]) for r in res["needles"]] == [tuple(t) for t in records_in]
        assert [[r["shard_mask"], r["damaged_bytes"], r["uncorrectable_bytes"]] for r in res["needles"]] == per
        check_invariants(res, k, res["needles"])


# ---------------------------------------------------------------------------------------------- volume images


def image(rng, dat_size, gaps=True, small_run=None):
    """A volume image of needle records after an 8-byte superblock: random sizes (a run of tiny ones at small_run),
    every fifth record deleted (in the image, not in the records), gaps between some.  Returns (dat, live records)."""
    dat = bytearray([3, 0, 0, 0, 0, 0, 0, 0])
    live, nid = [], 1
    while True:
        tiny = small_run is not None and small_run <= len(dat) < small_run + 4096
        n = int(rng.integers(0, 40)) if tiny else int(rng.integers(0, 3000))
        rec = no.write_record(nid, rng.integers(0, 256, n, dtype=np.uint8).tobytes(), append_at_ns=nid)
        if len(dat) + len(rec) > dat_size:
            break
        size = int.from_bytes(rec[12:16], "big")
        if nid % 5:
            live.append((nid, len(dat), size))
        dat += rec
        nid += 1
        if gaps and rng.random() < 0.1:
            dat += bytes(8 * int(rng.integers(1, 20)))
    dat += rng.integers(0, 256, dat_size - len(dat), dtype=np.uint8).tobytes()
    return np.frombuffer(bytes(dat), dtype=np.uint8).copy(), live


def device_run(swec, torch, shards, k, m, dat_size, large, small, records, radius=1):
    ec = swec.erasure_coding
    enc = ec.Encoder(k, m, device=0)
    dev = [torch.from_numpy(s).cuda() for s in shards]
    before = [d.clone() for d in dev]
    res = enc.locate_needle_damage_device([d.data_ptr() for d in dev], len(shards[0]), dat_size, records, radius=radius,
                                          large_block=large, small_block=small)
    assert all(torch.equal(x, y) for x, y in zip(dev, before))   # only read
    enc.close()
    return res


# ---------------------------------------------------------------------------------------------- CPU


def host_map_library(tmp_path):
    src = tmp_path / "stripe.cc"
    src.write_text('#include "%s"\n' % os.path.join(ROOT, "seaweedfs_b200", "csrc", "stripe_map.h") + r'''
extern "C" void map_all(int locate, int64_t size, int k, int64_t large, int64_t small, int64_t shard_len, int64_t* out) {
    const swec::StripeMap m = locate ? swec::StripeMap::locate(size, k, large, small) : swec::StripeMap::encode(size, k, large, small);
    for (int i = 0; i < k; i++)
        for (int64_t x = 0; x < shard_len; x++) out[i * shard_len + x] = m.dat_offset(i, x);
}
''')
    so = str(tmp_path / "libstripe.so")
    subprocess.run(["c++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"), "-o", so,
                    str(src)], check=True)
    L = C.CDLL(so)
    L.map_all.argtypes = [C.c_int, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_void_p]
    return L


def forward_map(k, dat_size, large, small):
    """Every data-shard byte's .dat offset (-1: padding), from the oracle's encode of an image whose bytes are the
    planes of (offset + 1)."""
    off = np.arange(1, dat_size + 1, dtype=np.int64)
    planes = [rn.encode_dat_image(((off >> (8 * p)) & 0xFF).astype(np.uint8), k, 1, large, small)[:k] for p in range(3)]
    n = len(planes[0][0])
    out = np.zeros((k, n), dtype=np.int64)
    for p, sh in enumerate(planes):
        out |= np.stack(sh).astype(np.int64) << (8 * p)
    return out - 1


GRID = [(k, large, small, size) for k, large, small in ((10, 10000, 100), (10, 4096, 512), (6, 3000, 1000), (3, 64, 8))
        for size in (0, 1, 8, small * k - 1, small * k, small * k + 1, large * k - 1, large * k, large * k + 1,
                     large * k + small * k, 2 * large * k + 3 * small * k, 2 * large * k + 3 * small * k + 17)]


@pytest.mark.parametrize("k,large,small,dat_size", GRID)
def test_host_inverse_striping_is_the_inverse_of_the_oracle(tmp_path, oracle, k, large, small, dat_size):
    """stripe_map.h's encode geometry, compiled for the host, against the oracle's forward striping, every byte of every
    data shard; and the plain walk used by the GPU tests agrees with both."""
    if dat_size == 0:
        assert rn.expected_shard_size(0, k, large, small) == 0
        return
    L = host_map_library(tmp_path)
    want = forward_map(k, dat_size, large, small)
    got = np.zeros_like(want)
    L.map_all(0, dat_size, k, large, small, want.shape[1], got.ctypes.data)
    assert np.array_equal(got, want)
    walk = Striping(k, dat_size, large, small)
    pick = np.random.default_rng(dat_size).integers(0, want.size, 200)
    assert all(walk(int(p) // want.shape[1], int(p) % want.shape[1]) == want.flat[p] for p in pick)


@pytest.mark.parametrize("k,large,small,dat_size", [(10, 10000, 100, 237_450), (10, 10000, 100, 100_000),
                                                    (6, 4096, 512, 3 * 4096 * 6 + 5000), (10, 1024, 64, 64_000)])
def test_host_inverse_striping_maps_locate_data_back_onto_each_record(tmp_path, swec, k, large, small, dat_size):
    """The locate geometry (the handle's reads): every LocateData interval of every record maps back onto the record."""
    L = host_map_library(tmp_path)
    shard_dat_size = dat_size // k
    n = rn.expected_shard_size(dat_size, k, large, small)
    got = np.zeros((k, n), dtype=np.int64)
    L.map_all(1, shard_dat_size, k, large, small, n, got.ctypes.data)
    _, records = image(np.random.default_rng(k + dat_size), dat_size)
    assert len(records) > 10
    for _, off, size in records:
        want = no.actual_size(size, 3)
        pos = off
        for iv in rn.locate_data(large, small, shard_dat_size, off, want, k):
            sid, soff = rn.interval_to_shard(iv, large, small, k)
            ln = iv[2]
            assert list(got[sid, soff:soff + ln]) == list(range(pos, pos + ln))
            pos += ln
        assert pos == off + want


def test_abi_struct_matches_the_header(swec):
    from seaweedfs_b200._native import NeedleDamage
    assert C.sizeof(NeedleDamage) == 40
    assert (NeedleDamage.shard_mask.offset, NeedleDamage.damaged_bytes.offset) == (20, 24)


def cpu_volume(tmp_path, k=10, m=4, name="5"):
    rng = np.random.default_rng(5)
    dat, live = image(rng, 300_000)
    base = str(tmp_path / name)
    for i, s in enumerate(rn.encode_dat_image(dat, k, m)):
        s.tofile(base + ".ec%02d" % i)
    open(base + ".ecx", "wb").write(rn.sorted_ecx_from_idx(b"".join(rn._entry(i, o // 8, s) for i, o, s in live)))
    json.dump({"version": 3, "datFileSize": str(len(dat)), "ecShardConfig": {"dataShards": k, "parityShards": m}},
              open(base + ".vif", "w"))
    return base


def raw_handle_call(swec, vol, radius=1, report=True, ranges_cap=0, needles_cap=0, needles=True, unowned=True):
    from seaweedfs_b200._native import DamageRange, DamageReport, NeedleDamage
    L = swec.lib()
    rep, n, nn, ok = DamageReport(), C.c_int(0), C.c_int(0), C.c_int(0)
    arr = (NeedleDamage * max(1, needles_cap))() if needles else None
    rng = (DamageRange * max(1, ranges_cap))()
    un = (C.c_uint64 * 2)() if unowned else None
    return L.swec_ec_volume_locate_needle_damage(vol._h, radius, C.byref(rep) if report else None, rng, ranges_cap,
                                                 C.byref(n), arr, needles_cap, C.byref(nn), un, C.byref(ok))


def test_argument_rules_and_their_order(swec, tmp_path):
    ec = swec.erasure_coding
    vol = ec.EcVolume(cpu_volume(tmp_path), device=-1)
    assert raw_handle_call(swec, vol, needles_cap=-1) == -1
    assert raw_handle_call(swec, vol, needles_cap=3, needles=False) == -1
    assert raw_handle_call(swec, vol, unowned=False) == -1
    # the new rules come first: a bad radius with them still names them
    assert raw_handle_call(swec, vol, radius=7, unowned=False) == -1
    assert b"unowned" in swec.lib().swec_last_error()
    assert raw_handle_call(swec, vol, radius=7) == -1 and b"radius" in swec.lib().swec_last_error()
    assert raw_handle_call(swec, vol, report=False) == -1
    assert raw_handle_call(swec, vol) == -7                      # every check passed: no device behind the handle
    vol.close()
    # device call: records NULL with n_records > 0, unowned NULL, both before the encoder is looked at
    from seaweedfs_b200._native import DamageReport
    L = swec.lib()
    rep, un = DamageReport(), (C.c_uint64 * 2)()
    args = [None, None, 4096, 1000, 10000, 100, 1, None, 3, C.byref(rep), None, 0, None]
    assert L.swec_locate_needle_damage_device(*args, un, None) == -1 and b"records" in L.swec_last_error()
    args[8] = 0
    assert L.swec_locate_needle_damage_device(*args, None, None) == -1 and b"unowned" in L.swec_last_error()
    assert L.swec_locate_needle_damage_device(*args, un, None) == -1             # NULL encoder
    enc = ec.Encoder(10, 4, device=-1)
    args[0], args[1] = enc._h, (C.c_void_p * 14)(*([1 << 20] * 14))
    args[6] = 3
    assert L.swec_locate_needle_damage_device(*args, un, None) == -1 and b"radius" in L.swec_last_error()
    args[6] = 1
    assert L.swec_locate_needle_damage_device(*args, un, None) == -7             # the device work is what fails
    enc.close()


def test_handle_file_checks(swec, tmp_path):
    ec = swec.erasure_coding
    base = cpu_volume(tmp_path)
    os.rename(base + ".ec12", base + ".ec12.away")
    vol = ec.EcVolume(base, device=-1)
    with pytest.raises(swec._native.SwecError) as e:
        vol.locate_needle_damage()
    assert e.value.status == -2 and ".ec12" in str(e.value)
    vol.close()
    os.rename(base + ".ec12.away", base + ".ec12")
    with open(base + ".ec03", "r+b") as f:
        f.truncate(os.path.getsize(base + ".ec03") - 1)
    vol = ec.EcVolume(base, device=-1)
    with pytest.raises(swec._native.SwecError) as e:
        vol.locate_needle_damage()
    assert e.value.status == -6
    vol.close()


def test_needle_damage_kernels_in_the_library(swec):
    """The __global__ functions of needle_damage.cu in libswec.so are exactly the one the GPU tests run."""
    from seaweedfs_b200 import _native
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("no CUDA toolkit")
    out = subprocess.run([cuobjdump, "-symbols", _native.library_path()], capture_output=True, text=True,
                         check=True).stdout
    syms = [ln.split()[-1] for ln in out.splitlines()
            if "STT_FUNC" in ln and "STO_ENTRY" in ln and "_needle_damage_cu_" in ln]
    assert [re.search(r"\d(nd_[a-z]+_kernel)E", s)[1] for s in syms] == ["nd_attribute_kernel"], syms
    assert not any(x in s for s in syms for x in ("_needles_cu_", "swec_locate_kernel", "rs10x4_encode", "swec_table"))


def test_locate_kernel_sass_is_unchanged(swec):
    """The locate kernels are untouched: every pinned swec_locate_kernel instantiation has its recorded SASS."""
    from seaweedfs_b200 import _native
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "locate_kernel_sass.json")))
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not (os.path.exists(cuobjdump) and os.path.exists(nvcc)):
        pytest.skip("no CUDA toolkit")
    if f"release {golden['nvcc_release']}," not in subprocess.run([nvcc, "--version"], capture_output=True,
                                                                  text=True).stdout:
        pytest.skip("the digests were taken with nvcc " + golden["nvcc_release"])
    out = subprocess.run([cuobjdump, "-sass", _native.library_path()], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s*Function : (\S+)\n", out)
    found = {}
    for name, body in zip(parts[1::2], parts[2::2]):
        mm = re.search(r"swec_locate_kernelILi(\d+)ELi(\d+)E", name)
        if mm:
            body = re.sub(r"_GLOBAL__N__\w+?_damage_cu_[0-9a-f]+", "", body.split("\n.....")[0]).strip()
            found[f"{mm.group(1)},{mm.group(2)}"] = hashlib.sha256(body.encode()).hexdigest()
    assert len(found) == 9
    for key, digest in golden["sha256"].items():
        assert found.get(key) == digest, key


# ---------------------------------------------------------------------------------------------- GPU: device level

K, M, LARGE, SMALL = 10, 4, 10000, 100
DAT = 2 * LARGE * K + 37 * SMALL * K + 450    # two large rows, small rows, a zero-padded tail row


def small_set(seed=1, k=K, m=M, dat_size=DAT, small_run=None):
    rng = np.random.default_rng(seed)
    dat, live = image(rng, dat_size, small_run=small_run)
    shards = rn.encode_dat_image(dat, k, m, LARGE, SMALL)
    return rng, dat, live, shards, Striping(k, dat_size, LARGE, SMALL)


def flip_dat(shards, walk, d, mask=0x5A):
    i, x = walk.shard_pos(d)
    shards[i][x] ^= np.uint8(mask)
    return i, x


SITES = ["superblock", "header", "data", "checksum", "padding", "two blocks", "one page", "deleted", "parity only"]


@pytest.mark.gpu
@pytest.mark.parametrize("site", SITES)
def test_device_sites(cuda, swec, site):
    rng, dat, live, shards, walk = small_set(small_run=150_000)
    rec = live[len(live) // 2]
    nid, off, size = rec
    end = off + no.actual_size(size, 3)
    named = None
    if site == "superblock":
        flip_dat(shards, walk, 3)
    elif site == "header":
        flip_dat(shards, walk, off + 13)
        named = nid
    elif site == "data":
        flip_dat(shards, walk, off + 20 + size // 3)
        named = nid
    elif site == "checksum":
        flip_dat(shards, walk, off + 16 + size + 1)
        named = nid
    elif site == "padding":
        flip_dat(shards, walk, end - 1)
        named = nid
    elif site == "two blocks":       # a record whose bytes lie in two blocks, so two shards
        nid, off, size = next(r for r in live if walk.shard_pos(r[1])[0] != walk.shard_pos(r[1] + no.actual_size(r[2], 3) - 1)[0])
        a = flip_dat(shards, walk, off)[0]
        b = flip_dat(shards, walk, off + no.actual_size(size, 3) - 1)[0]
        assert a != b
        named = nid
    elif site == "one page":         # many tiny records inside one 4 KiB page
        tiny = [r for r in live if 150_000 <= r[1] < 150_000 + 4096]
        assert len(tiny) > 20
        for r in tiny[::3]:
            flip_dat(shards, walk, r[1] + 1)
    elif site == "deleted":
        live_offs = {r[1] for r in live}
        d = 8
        while d in live_offs or Owners(live)(d) >= 0:
            d += 8
        flip_dat(shards, walk, d)
    else:
        shards[K + 1][123] ^= 7
        shards[K + 3][5000] ^= 1
    res = device_run(swec, cuda, shards, K, M, DAT, LARGE, SMALL, live)
    want = expected(shards, K, M, 1, live, walk)
    compare(res, want, live, K)
    hit = {r["needle_id"] for r in res["needles"] if r["damaged_bytes"] or r["uncorrectable_bytes"]}
    if named is not None:
        assert hit == {named}
    if site in ("superblock", "deleted"):
        assert hit == set() and res["unowned"] == [1, 0]
    if site == "parity only":
        assert hit == set() and res["unowned"] == [0, 0] and res["damaged_columns"] == 2
    if site == "one page":
        assert len(hit) == len([r for r in live if 150_000 <= r[1] < 150_000 + 4096][::3])


@pytest.mark.gpu
def test_zero_padded_tail_is_unowned(cuda, swec):
    _, _, live, shards, walk = small_set(seed=2)
    n = len(shards[0])
    shards[K - 1][n - 1] ^= 1              # padding of the tail row in the last data shard
    res = device_run(swec, cuda, shards, K, M, DAT, LARGE, SMALL, live)
    compare(res, expected(shards, K, M, 1, live, walk), live, K)
    assert res["unowned"] == [1, 0] and walk(K - 1, n - 1) == -1


@pytest.mark.gpu
def test_overlapping_damage_radius_1_then_2(cuda, swec):
    _, _, live, shards, walk = small_set(seed=3)
    nid, off, size = live[40]
    i, x = walk.shard_pos(off + 20)
    j = (i + 1) % K
    shards[i][x] ^= 0x11
    shards[j][x] ^= 0x22
    r1 = device_run(swec, cuda, shards, K, M, DAT, LARGE, SMALL, live, radius=1)
    compare(r1, expected(shards, K, M, 1, live, walk), live, K)
    assert r1["uncorrectable_columns"] == 1
    assert next(r for r in r1["needles"] if r["needle_id"] == nid)["uncorrectable_bytes"] >= 1
    r2 = device_run(swec, cuda, shards, K, M, DAT, LARGE, SMALL, live, radius=2)
    compare(r2, expected(shards, K, M, 2, live, walk), live, K)
    assert r2["uncorrectable_columns"] == 0 and sum(r["damaged_bytes"] for r in r2["needles"]) + r2["unowned"][0] == 2


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,radius", [(10, 4, 1), (10, 4, 2), (6, 3, 1), (20, 12, 1)])
def test_random_density_every_record(cuda, swec, k, m, radius):
    """Random damage at one density, one to three shards per damaged column: every record's counts."""
    dat_size = 2 * LARGE * k + 11 * SMALL * k + 77
    rng, dat, live, shards, walk = small_set(seed=10 + k, k=k, m=m, dat_size=dat_size)
    n = len(shards[0])
    cols = rng.choice(n, size=n // 150, replace=False)
    for c in cols:
        for sid in rng.choice(k + m, size=int(rng.integers(1, 4)), replace=False):
            shards[int(sid)][c] ^= np.uint8(rng.integers(1, 256))
    res = device_run(swec, cuda, shards, k, m, dat_size, LARGE, SMALL, live, radius=radius)
    want = expected(shards, k, m, radius, live, walk)
    compare(res, want, live, k)
    assert res["uncorrectable_columns"] > 0 and sum(r["damaged_bytes"] for r in res["needles"]) > 0


@pytest.mark.gpu
def test_overlapping_records(cuda, swec):
    """A corrupt index: records that overlap (and one repeated).  Every byte counts once, for the record with the
    greatest offset not above it."""
    _, _, live, shards, walk = small_set(seed=4)
    recs = list(live[:60])
    recs.append((9001, recs[10][1] + 8, recs[10][2] + 200))   # starts inside record 10 and runs past it
    recs.append((9002, recs[20][1], recs[20][2]))              # the same offset as record 20: the later entry wins
    for r in (recs[10], recs[20], recs[-2]):
        flip_dat(shards, walk, r[1] + 9)
        flip_dat(shards, walk, r[1] + no.actual_size(r[2], 3) - 2)
    res = device_run(swec, cuda, shards, K, M, DAT, LARGE, SMALL, recs)
    compare(res, expected(shards, K, M, 1, recs, walk), recs, K)
    by_id = {r["needle_id"]: r for r in res["needles"]}
    assert by_id[9002]["damaged_bytes"] == 2 and by_id[recs[20][0]]["damaged_bytes"] == 0


@pytest.mark.gpu
def test_damage_straddling_the_256_mib_piece(cuda, swec):
    """Shards of 256 MiB + 3 MiB: damage on both sides of the device piece, blamed and uncorrectable, against the
    analytic expectation (single-shard damage is blamed, two shards at radius 1 are uncorrectable)."""
    torch = cuda
    ec = swec.erasure_coding
    L = swec.lib()
    n = PIECE + 3 * MIB
    dat_size = K * n
    shards = [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(K + M)]
    for i in range(K):
        swec._native.check(L.swec_synth_fill_device(0, shards[i].data_ptr(), i * n, n, SEED, None))
    enc = ec.Encoder(K, M, device=0)
    enc.encode_device([s.data_ptr() for s in shards[:K]], [s.data_ptr() for s in shards[K:]], n)
    enc.synchronize()
    rng = np.random.default_rng(7)
    records, o = [], 8
    while o < dat_size:
        size = int(rng.integers(0, 5_000_000))
        records.append((len(records) + 1, o, size))
        o += no.actual_size(size, 3) + 8 * int(rng.integers(0, 3))
    walk = Striping(K, dat_size, GIB, MIB)
    flips = [(3, PIECE - 2), (3, PIECE - 1), (3, PIECE), (3, PIECE + 1), (0, 5)]
    for i, x in flips:
        shards[i][x] ^= 0x33
    shards[12][PIECE + 7] ^= 1
    unc = [PIECE - 9, PIECE + 9]
    for x in unc:
        shards[1][x] ^= 0x44
        shards[8][x] ^= 0x55
    torch.cuda.synchronize()
    res = enc.locate_needle_damage_device([s.data_ptr() for s in shards], n, dat_size, records, large_block=GIB,
                                          small_block=MIB)
    owner = Owners(records)
    per = {}
    unowned = [0, 0]

    def add(i, x, kind):
        j = owner(walk(i, x))
        if j < 0:
            unowned[kind] += 1
        else:
            e = per.setdefault(j, [0, 0, 0])
            e[0] |= 1 << i
            e[1 + kind] += 1
    for i, x in flips:
        add(i, x, 0)
    for x in unc:
        for i in range(K):
            add(i, x, 1)
    assert res["damaged_columns"] == len(flips) + 1 + len(unc) and res["uncorrectable_columns"] == len(unc)
    assert res["shards"] == {0: (1, 5, 5), 3: (4, PIECE - 2, PIECE + 1), 12: (1, PIECE + 7, PIECE + 7)}
    assert res["unowned"] == unowned
    got = {j: [r["shard_mask"], r["damaged_bytes"], r["uncorrectable_bytes"]] for j, r in enumerate(res["needles"])
           if r["damaged_bytes"] or r["uncorrectable_bytes"]}
    assert got == per
    check_invariants(res, K, res["needles"])
    del shards
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------- GPU: mounted volume


def generated_volume(swec, tmp_path, name, k=10, m=4, seed=20, dat_size=3_000_000, dat=None, live=None):
    """.dat + .idx written and EC-encoded by swec_ec_shards_generate (ratio from .vif when not 10+4)."""
    base = str(tmp_path / name)
    if dat is None:
        dat, live = image(np.random.default_rng(seed), dat_size, small_run=400_000)
    dat.tofile(base + ".dat")
    open(base + ".idx", "wb").write(b"".join(rn._entry(i, o // 8, s) for i, o, s in live))
    if (k, m) != (10, 4):
        json.dump({"ecShardConfig": {"dataShards": k, "parityShards": m}}, open(base + ".vif", "w"))
    swec.erasure_coding.volume_ec_shards_generate(base, needle_version=3)
    return base, dat, live


def handle_expected(base, k, m, radius, live, shard_dat_size):
    """The oracle over the shard files as they are, mapped through LocateData (the handle's reads)."""
    shards = [np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) for i in range(k + m)]
    pos = {}
    for j, (_, off, size) in enumerate(live):
        d = off
        for iv in rn.locate_data(GIB, MIB, shard_dat_size, off, no.actual_size(size, 3), k):
            sid, soff = rn.interval_to_shard(iv, GIB, MIB, k)
            ln = iv[2]
            pos[sid] = pos.get(sid, []) + [(soff, ln, d)]
            d += ln
    for v in pos.values():
        v.sort()
    starts = {s: [b[0] for b in v] for s, v in pos.items()}

    def dat_offset(i, x):          # -1 where no record lies: the owner walk then counts it as unowned
        j = bisect.bisect_right(starts.get(i, []), x) - 1
        if j < 0:
            return -1
        s, ln, d = pos[i][j]
        return d + x - s if x - s < ln else -1
    return expected(shards, k, m, radius, live, dat_offset)


def flip_file(path, off, mask=0x40):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)[0]
        f.seek(off)
        f.write(bytes([b ^ mask]))


def handle_compare(res, want, live, k=10):
    rep, per, unowned = want
    assert {key: res[key] for key in rep} == rep
    assert res["unowned"] == unowned
    hit = [(live[j], p) for j, p in enumerate(per) if p[1] or p[2]]
    hit.sort(key=lambda t: t[0][0])
    assert res["n_needles"] == len(hit)
    assert [(r["needle_id"], r["offset"], r["size"], [r["shard_mask"], r["damaged_bytes"], r["uncorrectable_bytes"]])
            for r in res["needles"]] == [(t[0][0], t[0][1], t[0][2], t[1]) for t in hit]
    check_invariants(res, k, res["needles"])


@pytest.mark.gpu
def test_handle_clean_set_does_no_second_pass(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    L = swec.lib()
    base, _, _ = generated_volume(swec, tmp_path, "1")
    ec.locate_ec_damage(base)                      # warm: the same kernels compiled / cached
    vol = ec.EcVolume(base)
    vol.locate_needle_damage()
    n0 = L.swec_kernel_launches()
    plain = ec.locate_ec_damage(base)
    n1 = L.swec_kernel_launches()
    res = vol.locate_needle_damage()
    n2 = L.swec_kernel_launches()
    assert n2 - n1 == n1 - n0 > 0
    assert res["ok"] and res["n_needles"] == 0 and res["needles"] == [] and res["unowned"] == [0, 0]
    assert {key: res[key] for key in plain} == plain
    vol.close()


@pytest.mark.gpu
def test_handle_scattered_damage_then_repair(cuda, swec, tmp_path):
    """Scattered damage: every needle named with its counts; the files are only read; then a repair restores exactly
    the needles without uncorrectable bytes, by the CRC check of scrub_needles."""
    ec = swec.erasure_coding
    base, dat, live = generated_volume(swec, tmp_path, "2")
    info = ec.EcVolume(base).info()
    walk = Striping(10, len(dat), GIB, MIB)
    rng = np.random.default_rng(3)
    for r in rng.choice(len(live), 25, replace=False):
        _, off, size = live[int(r)]
        flip_file(base + ".ec%02d" % walk.shard_pos(off + 20 + size // 2)[0],
                  walk.shard_pos(off + 20 + size // 2)[1], int(rng.integers(1, 256)))
    planted = set()
    for r in rng.choice(len(live), 4, replace=False):   # uncorrectable: two data shards of one column, inside Data
        nid, off, size = live[int(r)]
        planted.add(nid)
        i, x = walk.shard_pos(off + 24)
        flip_file(base + ".ec%02d" % i, x, 0x21)
        flip_file(base + ".ec%02d" % ((i + 3) % 10), x, 0x12)
    flip_file(base + ".ec11", 4321)                     # parity alone
    paths = [base + ".ec%02d" % i for i in range(14)]
    for p in paths:
        os.utime(p, ns=(10**18, 10**18))
    snap = {p: (open(p, "rb").read(), os.stat(p).st_mtime_ns) for p in paths}
    vol = ec.EcVolume(base)
    res = vol.locate_needle_damage()
    assert {p: (open(p, "rb").read(), os.stat(p).st_mtime_ns) for p in paths} == snap
    want = handle_expected(base, 10, 4, 1, live, info["shard_dat_size"])
    handle_compare(res, want, live)
    assert res["uncorrectable_columns"] > 0 and not res["ok"]
    lost = {r["needle_id"] for r in res["needles"] if r["uncorrectable_bytes"]}
    assert len(lost) >= 1
    ec.repair_ec_damage(base)
    _, _, errors = vol.scrub_needles(7)
    bad = {int(re.match(r"needle (\d+) on volume", e)[1]) for e in errors if e.startswith("needle ")}
    # every needle without uncorrectable bytes was restored; an uncorrectable column puts all k of its data bytes at
    # risk, so the needles named lost include neighbours whose own bytes in it happen to be intact
    assert bad <= lost and planted <= bad
    vol.close()


@pytest.mark.gpu
def test_handle_deleted_needles_and_the_cap(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    base, dat, live = generated_volume(swec, tmp_path, "3", seed=21)
    walk = Striping(10, len(dat), GIB, MIB)
    hit = live[5:15]
    for _, off, size in hit:
        i, x = walk.shard_pos(off + 17)
        flip_file(base + ".ec%02d" % i, x)
    vol = ec.EcVolume(base)
    gone = [hit[2][0], hit[7][0]]
    for nid in gone:
        vol.delete_needle(nid)
    res = vol.locate_needle_damage()
    kept = [r for r in live if r[0] not in gone]
    handle_compare(res, handle_expected(base, 10, 4, 1, kept, vol.info()["shard_dat_size"]), kept)
    assert res["n_needles"] == 8 and res["unowned"] == [2, 0]
    capped = vol.locate_needle_damage(max_needles=3)
    assert capped["n_needles"] == 8 and capped["needles"] == res["needles"][:3]
    vol.close()


@pytest.mark.gpu
def test_handle_vif_ratio_6_3(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    base, dat, live = generated_volume(swec, tmp_path, "4", k=6, m=3, seed=22)
    vol = ec.EcVolume(base)
    assert vol.info()["data_shards"] == 6
    walk = Striping(6, len(dat), GIB, MIB)
    for _, off, size in live[3:30:4]:
        i, x = walk.shard_pos(off + 30)
        flip_file(base + ".ec%02d" % i, x)
    res = vol.locate_needle_damage()
    handle_compare(res, handle_expected(base, 6, 3, 1, live, vol.info()["shard_dat_size"]), live, k=6)
    assert res["n_needles"] == 7
    vol.close()


@pytest.mark.gpu
def test_handle_reference_fixture(cuda, swec, tmp_path):
    if not os.path.exists(REF_DAT):
        pytest.skip("oracle/_ref/1.dat was not built")
    ec = swec.erasure_coding
    base = str(tmp_path / "1")
    shutil.copy(REF_DAT, base + ".dat")
    shutil.copy(REF_IDX, base + ".idx")
    ec.volume_ec_shards_generate(base)
    vol = ec.EcVolume(base)
    info = vol.info()
    live = [(k, o * 8, s) for k, o, s in rn._entries(open(REF_IDX, "rb").read())]
    byid = {}
    for k, o, s in live:
        byid[k] = (k, o, s)
    live = [r for r in byid.values() if r[2] > 0]
    walk = Striping(10, os.path.getsize(REF_DAT), GIB, MIB)
    for _, off, size in live[::3]:
        i, x = walk.shard_pos(off + 16)
        flip_file(base + ".ec%02d" % i, x)
    res = vol.locate_needle_damage()
    ecx = rn._entries(open(base + ".ecx", "rb").read())
    live_ecx = [(k, o * 8, s) for k, o, s in ecx if s > 0]
    handle_compare(res, handle_expected(base, 10, 4, 1, live_ecx, info["shard_dat_size"]), live_ecx)
    assert res["n_needles"] == len(live[::3])
    vol.close()


@pytest.mark.gpu
def test_handle_volume_just_over_one_large_row(cuda, swec, tmp_path):
    """10 GiB + 5 MiB: records around the seam between the large row and the small rows."""
    need = 10 * GIB * 2.6
    if shutil.disk_usage(str(tmp_path)).free < need:
        pytest.skip(f"needs {need / GIB:.0f} GiB free under {tmp_path}")
    ec = swec.erasure_coding
    base = str(tmp_path / "9")
    dat_size = 10 * GIB + 5 * MIB
    seam = 10 * GIB
    rng = np.random.default_rng(9)
    live, blobs, o = [], [], seam - 3 * MIB
    while o < dat_size - 300_000:
        n = int(rng.integers(0, 200_000))
        rec = no.write_record(len(live) + 1, rng.integers(0, 256, n, dtype=np.uint8).tobytes())
        live.append((len(live) + 1, o, int.from_bytes(rec[12:16], "big")))
        blobs.append((o, rec))
        o += len(rec)
    with open(base + ".dat", "wb") as f:
        f.write(bytes([3, 0, 0, 0, 0, 0, 0, 0]))
        f.truncate(dat_size)
        for off, rec in blobs:
            f.seek(off)
            f.write(rec)
    open(base + ".idx", "wb").write(b"".join(rn._entry(i, o // 8, s) for i, o, s in live))
    ec.volume_ec_shards_generate(base, needle_version=3)
    os.remove(base + ".dat")
    walk = Striping(10, dat_size, GIB, MIB)
    named = [live[j] for j in (0, len(live) // 2, len(live) - 1)]
    straddle = next(r for r in live if r[1] < seam < r[1] + no.actual_size(r[2], 3))
    named.append(straddle)
    for _, off, size in named:
        i, x = walk.shard_pos(off + 20)
        flip_file(base + ".ec%02d" % i, x)
    i, x = walk.shard_pos(straddle[1] + no.actual_size(straddle[2], 3) - 1)
    flip_file(base + ".ec%02d" % i, x)
    vol = ec.EcVolume(base)
    res = vol.locate_needle_damage()
    assert res["damaged_columns"] == 5 and res["uncorrectable_columns"] == 0
    by_id = {r["needle_id"]: r for r in res["needles"]}
    assert sorted(by_id) == sorted({r[0] for r in named})
    assert by_id[straddle[0]]["damaged_bytes"] == 2 and res["unowned"] == [0, 0]
    vol.close()
