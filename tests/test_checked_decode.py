"""The checked decode: swec_ec_shards_to_volume_checked (a whole EC volume), swec_write_dat_file_checked (shard files to
a .dat) and swec_decode_data_checked_device (shards in HBM).  Any k of the k+m shards decode the volume; damage the
check shards locate in the data shards is corrected before the .dat is written, and damage that cannot be corrected
fails the call with SWEC_ERR_UNCORRECTABLE and leaves neither .dat nor .idx.

The oracle is tests/damage_oracle.py's errors-and-erasures decoder (decode_columns with a presence mask), built on
oracle.rs_numpy: located errors of the information set are corrected, then R = G[lost]·G[I]^-1 rebuilds the lost data
shards.  Shard files come from the C oracle (encode_dat_image) or from swec_ec_shards_generate.

cpu: argument rules of the three calls; every file check of the volume call before device work, in order, with no .dat
or .idx left; the data shards alone need no GPU and give the plain call's .dat and .idx; the new status has a name and a
text; the SASS of every locate-kernel instantiation that existed before the decoding mode is unchanged.
gpu: device level, one wrong byte of every value at every present position of RS(10,4) with nothing, every single
shard and a sample of two shards lost, and two wrong shards in a column past the radius; file level, a needle volume
with scattered damage in several data shards and 0, 1 or 2 shards lost, against the damaged .dat the plain call writes;
uncorrectable columns; radius 0; large rows, small rows and the ragged tail with small blocks, slot boundaries, a 6+3
ratio from .vif, a shard in an additional directory and O_DIRECT."""
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

from oracle import rs_numpy as rn  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAST_NS = 1_000_000_000 * 1_000_000_000    # an mtime no write can produce


# ---------------------------------------------------------------------------------------------- helpers


def needle_volume(seed=11, needles=120, version=3):
    """A well-formed volume image: 8-byte superblock (byte 0 = needle version), 8-byte aligned needle records, and the
    .idx that indexes them, with overwrites and deletions."""
    rng = np.random.default_rng(seed)
    dat = bytearray([version, 0, 0, 0, 0, 0, 0, 0])
    idx = b""
    for _ in range(needles):
        key = int(rng.integers(1, max(2, needles // 2)))
        size = int(rng.integers(1, 40000))
        fixed = 16 + size + 4 + (8 if version == 3 else 0)
        offset = len(dat) // 8
        dat += rng.integers(0, 256, fixed + (8 - fixed % 8), dtype=np.uint8).tobytes()
        idx += rn._entry(key, offset, rn.TOMBSTONE if int(rng.integers(0, 12)) == 0 else size)
    return np.frombuffer(bytes(dat), dtype=np.uint8).copy(), idx


def lay_down(oracle, tmp_path, dat, idx, k=10, m=4, name="7", vif=True):
    """What a finished ec.encode leaves on disk, written by the C oracle (production block sizes)."""
    base = str(tmp_path / name)
    shards = oracle.encode_dat_image(dat, k=k, m=m)
    for i, s in enumerate(shards):
        s.tofile(base + ".ec%02d" % i)
    open(base + ".ecx", "wb").write(rn.sorted_ecx_from_idx(idx))
    if vif:
        json.dump({"version": int(dat[0]), "datFileSize": str(len(dat)),
                   "ecShardConfig": {"dataShards": k, "parityShards": m}}, open(base + ".vif", "w"))
    return base, shards


def paths(base, n=14):
    return [base + ".ec%02d" % i for i in range(n) if os.path.exists(base + ".ec%02d" % i)]


def snapshot(ps):
    return {p: (open(p, "rb").read(), os.stat(p).st_mtime_ns) for p in ps}


def age(ps):
    for p in ps:
        os.utime(p, ns=(PAST_NS, PAST_NS))


def flip(path, off, mask=0x40):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ mask]))


def no_outputs(base):
    return not os.path.exists(base + ".dat") and not os.path.exists(base + ".idx")


def mask(n, lost):
    return tuple(i not in lost for i in range(n))


def checked_decode(shards, k, m, present, radius=1):
    """What the checked decode gives for the shards (lost ones may be None): (the k data shards, report)."""
    info, checks, lost, _, r = do.punctured_rows(k, m, present)
    length = len(shards[info[0]])
    x = [shards[i].copy() for i in info]
    c = len(checks)
    if c == 0:
        rep = {"ok": False, "columns": 0, "damaged_columns": 0, "uncorrectable_columns": 0, "first_uncorrectable": -1,
               "last_uncorrectable": -1, "shards": {}, "ranges": [], "n_ranges": 0}
    else:
        cols, a, b, va, vb, ids = do.decode_columns(shards, k, m, min(radius, c // 2), present)
        for pa, ev in ((a, va), (b, vb)):       # errors of information positions come out before R rebuilds
            for j in range(k):
                sel = pa == j
                x[j][cols[sel]] ^= ev[sel]
        ida = np.where(a >= 0, ids[np.maximum(a, 0)], -1)
        idb = np.where(b >= 0, ids[np.maximum(b, 0)], -1)
        rep = do.report(length, k + m, cols, ida, idb)
        rep["ok"] = rep["uncorrectable_columns"] == 0
    data = {i: x[j] for j, i in enumerate(info) if i < k}
    data.update({i: v for i, v in zip(lost, rn.apply_rows(r, x)) if i < k})
    return [data[i] for i in range(k)], rep


# ------------------------------------------------------------------------------------------ CPU


def _file_call(L, base, names, k=10, m=4, radius=1, report=True, cap=4, ranges=True, ok=True, device=-1, size=1000):
    from seaweedfs_b200._native import DamageRange, DamageReport
    rep, rng_arr, n, okv = DamageReport(), (DamageRange * 4)(), C.c_int(0), C.c_int(7)
    arr = (C.c_char_p * len(names))(*[p.encode() if p else None for p in names]) if names is not None else None
    rc = L.swec_write_dat_file_checked(base.encode(), size, arr, k, m, 10000, 100, device, radius,
                                       C.byref(rep) if report else None, rng_arr if ranges else None, cap, C.byref(n),
                                       C.byref(okv) if ok else None)
    return rc, okv.value


def test_checked_decode_argument_rules(swec, oracle, tmp_path):
    from seaweedfs_b200._native import DamageRange, DamageReport
    ec = swec.erasure_coding
    L = swec.lib()
    rng = np.random.default_rng(1)
    shards = [rng.integers(0, 256, 1000, dtype=np.uint8) for _ in range(10)]
    shards += rn.encode(10, 4, shards)
    base = str(tmp_path / "6")
    for i, s in enumerate(shards):
        s.tofile(base + ".ec%02d" % i)
    names = [base + ".ec%02d" % i for i in range(14)]
    names[3] = None
    age(paths(base))
    before = snapshot(paths(base))
    for kw in ({"radius": -1}, {"radius": 3}, {"report": False}, {"cap": -1}, {"ranges": False}, {"ok": False},
               {"names": None}, {"k": 0}, {"m": 0}, {"k": 30, "m": 3}):
        rc, okv = _file_call(L, base, kw.pop("names", names), **kw)
        assert rc == -1, kw
        assert not os.path.exists(base + ".dat"), kw
    assert _file_call(L, base, names, radius=3)[0] == -1 and b"radius must be 0, 1 or 2" in L.swec_last_error()
    for radius in (0, 1, 2):                               # valid: on to the device, whose absence removes the .dat
        assert _file_call(L, base, names, radius=radius) == (-7, 0)
        assert not os.path.exists(base + ".dat")
    assert _file_call(L, base, names, ranges=False, cap=0) == (-7, 0)
    assert snapshot(paths(base)) == before

    rep, rng_arr, n, okv, size = DamageReport(), (DamageRange * 4)(), C.c_int(0), C.c_int(0), C.c_int64(0)
    for kw in ({"radius": -1}, {"radius": 3}, {"report": None}, {"ok": None}, {"cap": -1}, {"ranges": None}):
        a = {"radius": 1, "report": C.byref(rep), "ok": C.byref(okv), "cap": 4, "ranges": rng_arr, **kw}
        assert L.swec_ec_shards_to_volume_checked(base.encode(), None, None, 0, -1, a["radius"], C.byref(size),
                                                  a["report"], a["ranges"], a["cap"], C.byref(n), a["ok"]) == -1, kw
    assert no_outputs(base)

    e104 = ec.Encoder(10, 4, device=-1)
    present = (C.c_uint8 * 14)(*([0] + [1] * 12 + [0]))
    ptrs = (C.c_void_p * 14)(*([1 << 20] * 13 + [None]))   # a missing parity shard needs no buffer

    def dev_call(radius=1, report=C.byref(rep), ranges=rng_arr, cap=4, pres=present, p=ptrs):
        return L.swec_decode_data_checked_device(e104._h, p, pres, 4096, radius, report, ranges, cap, C.byref(n), None)

    for kw in ({"radius": -1}, {"radius": 3}, {"report": None}, {"cap": -1}, {"ranges": None}, {"pres": None},
               {"p": None}):
        assert dev_call(**kw) == -1, kw
    assert dev_call(p=(C.c_void_p * 14)(*([None] + [1 << 20] * 13))) == -1     # the data shard to rebuild has none
    assert b"missing shard has no buffer" in L.swec_last_error()
    assert dev_call(p=(C.c_void_p * 14)(*([1 << 20] * 5 + [None] + [1 << 20] * 8))) == -1   # a present data shard
    assert dev_call(p=(C.c_void_p * 14)(*([1 << 20] * 11 + [None] + [1 << 20] * 2))) == -1  # a present parity shard
    assert dev_call(pres=(C.c_uint8 * 14)(*([0] * 5 + [1] * 9))) == -2
    for radius in (0, 1, 2):
        assert dev_call(radius=radius) == -7
    assert dev_call(ranges=None, cap=0) == -7
    with pytest.raises(swec.SwecError) as e:
        e104.decode_data_checked_device([1 << 20] * 13 + [None], [0] + [1] * 12 + [0], 4096)
    assert e.value.name == "SWEC_ERR_NO_DEVICE"


def _expect_failure(swec, base, name, text=None, **kw):
    with pytest.raises(swec.SwecError) as e:
        swec.erasure_coding.ec_shards_to_volume_checked(base, device=-1, **kw)
    assert e.value.name == name, str(e.value)
    if text:
        assert text in str(e.value), str(e.value)
    assert no_outputs(base)


def test_every_file_check_comes_before_device_work(swec, oracle, tmp_path):
    dat, idx = needle_volume(seed=3, needles=60)
    base, shards = lay_down(oracle, tmp_path, dat, idx, vif=False)
    ecj = b"".join(key.to_bytes(8, "big") for key, _, _ in list(rn._entries(rn.sorted_ecx_from_idx(idx)))[:2])
    open(base + ".ecj", "wb").write(ecj)
    ecx = open(base + ".ecx", "rb").read()
    age(paths(base))
    before = snapshot(paths(base))

    for i in (1, 4, 7, 11, 13):                           # too few shards: 9 of 14
        os.rename(base + ".ec%02d" % i, base + ".x%02d" % i)
    _expect_failure(swec, base, "SWEC_ERR_TOO_FEW_SHARDS", "has 9 of its 14 shards, needs at least 10")
    for i in (1, 4, 7, 11, 13):
        os.rename(base + ".x%02d" % i, base + ".ec%02d" % i)
    # .ec00 missing and no .vif: the needle version is unknown, and nothing is written (the .ecj is not folded)
    os.rename(base + ".ec00", base + ".x00")
    _expect_failure(swec, base, "SWEC_ERR_TOO_FEW_SHARDS", "no .ec00 and no needle version in its .vif")
    assert open(base + ".ecx", "rb").read() == ecx and os.path.exists(base + ".ecj")
    os.rename(base + ".x00", base + ".ec00")
    assert snapshot(paths(base)) == before

    with open(base + ".ec12", "ab") as f:                 # unequal lengths
        f.write(b"x")
    _expect_failure(swec, base, "SWEC_ERR_SHARD_SIZE", "ec shard size expected %d actual %d" % (len(shards[0]),
                                                                                               len(shards[0]) + 1))
    os.truncate(base + ".ec12", len(shards[0]))
    for i in range(14):                                   # every shard shorter than the copy plan needs
        os.truncate(base + ".ec%02d" % i, 1000)
    _expect_failure(swec, base, "SWEC_ERR_IO", "short read copying shard 0")
    for i in range(14):
        shards[i].tofile(base + ".ec%02d" % i)

    keys = [key for key, _, _ in rn._entries(rn.sorted_ecx_from_idx(idx))]
    open(base + ".ecj", "wb").write(b"".join(key.to_bytes(8, "big") for key in keys))
    _expect_failure(swec, base, "SWEC_ERR_NO_LIVE_NEEDLES", "no live entries")
    assert not os.path.exists(base + ".ecj")                # folded before the live check, as the plain call does

    base2, _ = lay_down(oracle, tmp_path, dat, idx, name="9")
    os.remove(base2 + ".ec00")                            # .vif has the version: on to the device, nothing left
    _expect_failure(swec, base2, "SWEC_ERR_NO_DEVICE")


def test_data_shards_alone_need_no_gpu(swec, oracle, tmp_path):
    ec = swec.erasure_coding
    dat, idx = needle_volume(seed=5, needles=200)
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    out = {}
    for d in ("a", "b"):
        base, _ = lay_down(oracle, tmp_path / d, dat, idx, k=6, m=3)
        for i in range(6, 9):
            os.remove(base + ".ec%02d" % i)
        open(base + ".ecj", "wb").write(next(rn._entries(rn.sorted_ecx_from_idx(idx)))[0].to_bytes(8, "big"))
        if d == "a":
            size = ec.volume_ec_shards_to_volume(base)
        else:
            res = ec.ec_shards_to_volume_checked(base, device=-1)
            size = res["dat_file_size"]
            assert res["ok"] is False and res["columns"] == 0 and res["damaged_columns"] == 0 and res["ranges"] == []
        out[d] = (size, open(base + ".dat", "rb").read(), open(base + ".idx", "rb").read())
    assert out["a"] == out["b"]
    assert out["a"][1] == dat[:out["a"][0]].tobytes()


def test_uncorrectable_status_has_a_name_and_a_text(swec):
    from seaweedfs_b200._native import STATUS
    L = swec.lib()
    assert STATUS[-12] == "SWEC_ERR_UNCORRECTABLE"
    assert L.swec_strerror(-12) == b"damage that cannot be corrected remains"
    header = open(os.path.join(ROOT, "include", "swec.h")).read()
    assert re.search(r"SWEC_ERR_UNCORRECTABLE = -12\b", header)


def _locate_kernel_sass(lib_path):
    out = subprocess.run([shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump", "-sass", lib_path],
                         capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s*Function : (\S+)\n", out)
    found = {}
    for name, body in zip(parts[1::2], parts[2::2]):
        m = re.search(r"swec_locate_kernelILi(\d+)ELi(\d+)E", name)
        if m:
            body = re.sub(r"_GLOBAL__N__\w+?_damage_cu_[0-9a-f]+", "", body.split("\n.....")[0]).strip()
            found[f"{m.group(1)},{m.group(2)}"] = hashlib.sha256(body.encode()).hexdigest()
    return found


def test_existing_locate_kernels_keep_their_sass(swec):
    """The decoding mode is a template instantiation of its own: the locate, correct and rebuild instantiations
    compile to the same SASS as before it existed."""
    from seaweedfs_b200 import _native
    golden = json.load(open(os.path.join(ROOT, "tests", "golden", "locate_kernel_sass.json")))
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not (os.path.exists(cuobjdump) and os.path.exists(nvcc)):
        pytest.skip("no CUDA toolkit")
    if f"release {golden['nvcc_release']}," not in subprocess.run([nvcc, "--version"], capture_output=True,
                                                                  text=True).stdout:
        pytest.skip("the digests were taken with nvcc " + golden["nvcc_release"])
    found = _locate_kernel_sass(_native.library_path())
    for key, digest in golden["sha256"].items():
        assert found.get(key) == digest, key
    assert {"0,3", "3,3", "4,3"} <= set(found)             # the decoding instantiations


# ------------------------------------------------------------------------------------------ GPU


def _device_case(ec, torch, enc, clean, present, radius, damaged):
    """swec_decode_data_checked_device on `damaged` (k+m numpy shards) with the lost ones given no data: (data after,
    parity after, report)."""
    k = 10
    bufs = [torch.from_numpy(s.copy()).cuda() if present[i] or i < k else None for i, s in enumerate(damaged)]
    for i in range(k):
        if not present[i]:
            bufs[i].fill_(0xA5)
    ptrs = [b.data_ptr() if b is not None else None for b in bufs]
    rep = enc.decode_data_checked_device(ptrs, [int(p) for p in present], len(clean[0]), radius=radius)
    torch.cuda.synchronize()
    return [b.cpu().numpy() if b is not None else None for b in bufs], rep


@pytest.mark.gpu
def test_device_every_single_error_with_erasures(cuda, swec):
    """One wrong byte of every value at every present position, for nothing lost, every single lost shard and a
    sample of two lost: every data buffer ends up equal to the original, present parity is untouched, and the report
    is the oracle's."""
    ec = swec.erasure_coding
    torch = cuda
    k, m = 10, 4
    enc = ec.Encoder(k, m)
    losses = [()] + [(i,) for i in range(14)] + [(0, 1), (2, 9), (4, 12), (10, 11), (0, 13), (7, 10)]
    for lost in losses:
        present = mask(14, lost)
        ids = [i for i in range(14) if present[i]]
        length = 255 * len(ids) + 5                        # a byte tail after the last whole vector
        rng = np.random.default_rng(len(lost) * 100 + sum(lost))
        clean = [rng.integers(0, 256, length, dtype=np.uint8) for _ in range(k)]
        clean += rn.encode(k, m, clean)
        damaged = [s.copy() for s in clean]
        for p, sid in enumerate(ids):
            damaged[sid][p * 255:(p + 1) * 255] ^= np.arange(1, 256, dtype=np.uint8)
        got, rep = _device_case(ec, torch, enc, clean, present, 1, damaged)
        for i in range(k):
            assert (got[i] == clean[i]).all(), (lost, i)
        for i in range(k, 14):
            if present[i]:
                assert (got[i] == damaged[i]).all(), (lost, i)
        want_data, want = checked_decode([d if present[i] else None for i, d in enumerate(damaged)], k, m, present)
        assert {"ok": rep["uncorrectable_columns"] == 0, **rep} == want, lost
        assert rep["damaged_columns"] == 255 * len(ids) and rep["uncorrectable_columns"] == 0, lost
        assert all((w == c).all() for w, c in zip(want_data, clean[:k]))


@pytest.mark.gpu
def test_device_two_wrong_shards_past_the_radius(cuda, swec):
    """c = 3 at radius 1: two wrong present shards in a column are reported, and the data bytes are those of
    swec_reconstruct_device(data_only=1) on the shards as found."""
    ec = swec.erasure_coding
    torch = cuda
    k, m = 10, 4
    enc = ec.Encoder(k, m)
    length = 40_000
    rng = np.random.default_rng(7)
    clean = [rng.integers(0, 256, length, dtype=np.uint8) for _ in range(k)]
    clean += rn.encode(k, m, clean)
    for lost in ((3,), (12,)):
        present = mask(14, lost)
        damaged = [s.copy() for s in clean]
        cols = np.sort(rng.choice(length, 300, replace=False))
        ids = [i for i in range(14) if present[i]]
        for x in cols:
            for sid in rng.choice(ids, 2, replace=False):
                damaged[int(sid)][x] ^= np.uint8(rng.integers(1, 256))
        one = np.setdiff1d(np.arange(0, length, 97), cols)[:100]   # and some single errors, corrected
        for x in one:
            damaged[int(rng.choice(ids))][x] ^= np.uint8(rng.integers(1, 256))
        got, rep = _device_case(ec, torch, enc, clean, present, 1, damaged)
        want_data, want = checked_decode([d if present[i] else None for i, d in enumerate(damaged)], k, m, present)
        assert {"ok": rep["uncorrectable_columns"] == 0, **rep} == want
        assert rep["uncorrectable_columns"] == len(cols) and rep["damaged_columns"] == len(cols) + len(one)
        # plain ReconstructData on the shards as found
        plain = [torch.from_numpy(d.copy()).cuda() for d in damaged]
        for i in lost:
            plain[i].zero_()
        enc.reconstruct_device([p.data_ptr() for p in plain], [int(p) for p in present], length, data_only=True)
        torch.cuda.synchronize()
        for i in range(k):
            assert (got[i] == want_data[i]).all(), i
            assert (got[i][cols] == plain[i].cpu().numpy()[cols]).all(), i
            assert (got[i][one] == clean[i][one]).all(), i


def _generate(swec, tmp_path, name="5", needles=1300, seed=21):
    """A needle volume encoded by swec_ec_shards_generate; the original .dat moved aside."""
    ec = swec.erasure_coding
    dat, idx = needle_volume(seed=seed, needles=needles)
    base = str(tmp_path / name)
    dat.tofile(base + ".dat")
    open(base + ".idx", "wb").write(idx)
    ec.volume_ec_shards_generate(base)
    os.remove(base + ".dat")
    os.remove(base + ".idx")
    return base, dat


def _scatter(base, shard_ids, columns, seed):
    """Flip one byte in each of `columns` columns, in a different column per flip, on the given shards in turn."""
    rng = np.random.default_rng(seed)
    size = os.path.getsize(base + ".ec00")
    offs = np.sort(rng.choice(size, columns, replace=False))
    for j, off in enumerate(offs):
        flip(base + ".ec%02d" % shard_ids[j % len(shard_ids)], int(off), int(rng.integers(1, 256)))
    return offs


def _read_shards(base, n=14):
    return [np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) if os.path.exists(base + ".ec%02d" % i) else None
            for i in range(n)]


@pytest.mark.gpu
def test_volume_decode_corrects_scattered_damage(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    base, dat = _generate(swec, tmp_path)
    assert len(dat) > 20 << 20                           # small rows and a tail row of 1 MiB blocks
    offs = _scatter(base, [0, 2, 5, 9], 400, 22)
    assert (offs >= 2 << 20).any()                       # damage in the tail row too
    age(paths(base))
    # the plain call copies the damage into the .dat
    plain_size = ec.volume_ec_shards_to_volume(base)
    plain_dat = np.fromfile(base + ".dat", dtype=np.uint8)
    plain_idx = open(base + ".idx", "rb").read()
    assert (plain_dat != dat[:plain_size]).sum() > 250
    os.remove(base + ".dat")
    os.remove(base + ".idx")
    for lost in ((), (3,), (1, 12), (11, 13)):
        aside = {}
        for i in lost:
            aside[i] = base + ".lost%02d" % i
            os.rename(base + ".ec%02d" % i, aside[i])
        before = snapshot(paths(base))
        shards = _read_shards(base)
        present = mask(14, lost)
        res = ec.ec_shards_to_volume_checked(base)
        assert res["dat_file_size"] == plain_size
        out = np.fromfile(base + ".dat", dtype=np.uint8)
        assert len(out) == plain_size and (out == dat[:plain_size]).all(), lost
        assert open(base + ".idx", "rb").read() == plain_idx
        cols = res["columns"]
        _, want = checked_decode([s[:cols] if s is not None else None for s in shards], 10, 4, present)
        assert {"dat_file_size": plain_size, **want} == res, lost
        assert res["ok"] and res["damaged_columns"] > 0
        assert snapshot(paths(base)) == before
        os.remove(base + ".dat")
        os.remove(base + ".idx")
        for i, p in aside.items():
            os.rename(p, base + ".ec%02d" % i)


@pytest.mark.gpu
def test_volume_decode_uncorrectable_and_radius_0(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    base, dat = _generate(swec, tmp_path, name="6", needles=200, seed=31)
    os.rename(base + ".ec02", base + ".lost")
    res = ec.ec_shards_to_volume_checked(base, radius=0)   # a clean set decodes at radius 0
    assert res["ok"] and res["damaged_columns"] == 0
    assert (np.fromfile(base + ".dat", dtype=np.uint8) == dat[:res["dat_file_size"]]).all()
    os.remove(base + ".dat")
    os.remove(base + ".idx")

    flip(base + ".ec07", 5000)                          # one wrong shard: radius 0 refuses, radius 1 corrects
    age(paths(base))
    before = snapshot(paths(base))
    with pytest.raises(swec.SwecError) as e:
        ec.ec_shards_to_volume_checked(base, radius=0)
    assert e.value.name == "SWEC_ERR_UNCORRECTABLE" and "no .dat written" in str(e.value)
    assert e.value.report["uncorrectable_columns"] == 1 and e.value.report["first_uncorrectable"] == 5000
    assert no_outputs(base)
    assert ec.ec_shards_to_volume_checked(base)["ok"]
    os.remove(base + ".dat")
    os.remove(base + ".idx")

    flip(base + ".ec09", 5000)                          # two wrong shards with c = 3: reported at radius 1
    flip(base + ".ec00", 77_777)
    flip(base + ".ec11", 77_777)
    shards = _read_shards(base)
    age(paths(base))
    before = snapshot(paths(base))
    with pytest.raises(swec.SwecError) as e:
        ec.ec_shards_to_volume_checked(base)
    assert e.value.name == "SWEC_ERR_UNCORRECTABLE"
    cols = e.value.report["columns"]
    _, want = checked_decode([s[:cols] if s is not None else None for s in shards], 10, 4, mask(14, (2,)))
    assert {"ok": False, **e.value.report} == want
    assert e.value.report["uncorrectable_columns"] == 2
    assert no_outputs(base)
    assert snapshot(paths(base)) == before


def _small_block_set(oracle, tmp_path, k, m, dat_size, seed, name="s"):
    rng = np.random.default_rng(seed)
    dat = rng.integers(0, 256, dat_size, dtype=np.uint8)
    shards = oracle.encode_dat_image(dat, k=k, m=m, buffer_size=100, large=10000, small=100)
    base = str(tmp_path / name)
    for i, s in enumerate(shards):
        s.tofile(base + ".ec%02d" % i)
    return base, dat, shards


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,lost", [(10, 4, ()), (10, 4, (0,)), (10, 4, (4, 13)), (6, 3, (5,)), (6, 3, ())])
def test_write_dat_file_checked_small_blocks(cuda, swec, oracle, tmp_path, monkeypatch, k, m, lost):
    """Large blocks of 10000 and small of 100 bytes: large rows, small rows several to a slot, and the ragged tail;
    a slot of 4 KiB cuts large rows and batches of small rows."""
    ec = swec.erasure_coding
    monkeypatch.setenv("SWEC_FILE_CHUNK", "4096")
    dat_size = 3 * k * 10000 + 57 * k * 100 + 3 * 100 + 37   # 3 large rows, 57 small rows, a tail over 4 shards
    base, dat, clean = _small_block_set(oracle, tmp_path, k, m, dat_size, seed=k * 10 + len(lost))
    rng = np.random.default_rng(5)
    size = len(clean[0])
    damaged = [s.copy() for s in clean]
    present = mask(k + m, lost)
    ids = [i for i in range(k) if present[i]]
    for j, x in enumerate(np.sort(rng.choice(size, 250, replace=False))):   # one wrong data byte per column
        sid = ids[j % len(ids)]
        damaged[sid][x] ^= np.uint8(rng.integers(1, 256))
        flip(base + ".ec%02d" % sid, int(x), int(damaged[sid][x] ^ clean[sid][x]))
    names = [base + ".ec%02d" % i if present[i] else None for i in range(k + m)]
    res = ec.write_dat_file_checked(str(tmp_path / "out"), dat_size, names, data_shards=k, parity_shards=m,
                                    large_block=10000, small_block=100)
    out = np.fromfile(str(tmp_path / "out.dat"), dtype=np.uint8)
    assert len(out) == dat_size and (out == dat).all()
    cols = 3 * 10000 + 57 * 100 + 100
    assert res["columns"] == cols and res["ok"]
    _, want = checked_decode([d[:cols] if present[i] else None for i, d in enumerate(damaged)], k, m, present)
    assert {"dat_file_size": dat_size, **want} == res
    if not lost:                                          # the plain call copies the damage
        ec.write_dat_file(str(tmp_path / "plain"), dat_size, names[:k], data_shards=k, large_block=10000,
                          small_block=100)
        assert (np.fromfile(str(tmp_path / "plain.dat"), dtype=np.uint8) != dat).sum() > 200


@pytest.mark.gpu
def test_volume_decode_ratio_from_vif_additional_dir_and_o_direct(cuda, swec, oracle, tmp_path):
    ec = swec.erasure_coding
    L = swec.lib()
    dat, idx = needle_volume(seed=41, needles=900)
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    base, shards = lay_down(oracle, tmp_path / "a", dat, idx, k=6, m=3)
    os.remove(base + ".ec00")                            # the version comes from .vif; c = 2 check shards
    for i in (3, 8):
        os.rename(base + ".ec%02d" % i, str(tmp_path / "b" / ("7.ec%02d" % i)))
    for sid, off in [(1, 1000), (3, 2_000_000), (5, 700_001), (4, 123)]:
        p = base + ".ec%02d" % sid if sid != 3 else str(tmp_path / "b" / "7.ec03")
        flip(p, off)
    assert L.swec_set_option(b"file_direct_io", 3) == 0
    try:
        res = ec.ec_shards_to_volume_checked(base, additional_dirs=[str(tmp_path / "b")])
    finally:
        assert L.swec_set_option(b"file_direct_io", int(os.environ.get("SWEC_FILE_DIRECT", "0")) & 3) == 0
    size = res["dat_file_size"]
    assert size == rn.find_dat_file_size(rn.sorted_ecx_from_idx(idx), 3)
    assert (np.fromfile(base + ".dat", dtype=np.uint8) == dat[:size]).all()
    assert res["ok"] and res["damaged_columns"] == 4
    assert res["shards"] == {1: (1, 1000, 1000), 3: (1, 2_000_000, 2_000_000), 4: (1, 123, 123),
                             5: (1, 700_001, 700_001)}
