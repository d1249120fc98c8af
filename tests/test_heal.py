"""The heal: swec_heal_device (shards in HBM), swec_heal_ec_files (shard files) and swec_ec_shards_heal (a whole EC
volume).  One decode of the code punctured to the present shards rebuilds the lost shards and corrects the damaged
present ones in place; a column it cannot decode within t = min(radius, c // 2) keeps its present bytes, and its
rebuilt bytes are plain rebuild's (include/swec.h).

The oracle is tests/damage_oracle.py's errors-and-erasures column decoder (decode_columns over error_table): the located
error values are XORed into their own positions' bytes, information and check alike, and R = G[lost]·G[I]^-1 rebuilds
the lost shards from the corrected information set.

cpu: the argument rules of the three calls, pinned to those of swec_reconstruct_checked_device,
swec_rebuild_ec_files_checked and swec_ec_shards_rebuild.
gpu: device level on RS(10,4), RS(6,3) and RS(12,8) with every number of lost shards at radius 0, 1 and 2, damage within
t, between t+1 and c-t and beyond c-t at the vector, warp-window, page and partial-vector seams, aligned and unaligned,
against the oracle, reconstruct_checked_device and (nothing lost) correct_damage_device; two 256 MiB pieces; file level
against the oracle, the checked rebuild and the checked rebuild followed by the repair; the column the two-call flow
rewrites into another codeword; untouched files keep their mtime; pass 2's pipeline reads only the flagged pages; a
failure leaves no rebuilt file; a second call finds nothing; the volume call folds the .ecj."""
import ctypes as C
import json
import os
import shutil

import numpy as np
import pytest

import damage_oracle as do
from oracle import rs_numpy as rn
from test_checked_decode import lay_down, needle_volume

PAST_NS = 1_000_000_000 * 1_000_000_000    # an mtime no write can produce
MIB = 1 << 20


def _set(L, **opts):
    for name, value in opts.items():
        assert L.swec_set_option(name.encode(), int(value)) == 0, (name, value)


@pytest.fixture(scope="module", autouse=True)
def inline_compiles(swec):
    """The shards here are short, so the applies of the loss patterns' matrices would queue their run-time kernels for
    the background compiler, which would still be compiling them while later modules run.  jit_min_bytes 0 compiles
    them inline at device level, and the file calls run with jit 0 (the file pipeline never waits for a compile); the
    documented defaults come back afterwards."""
    L = swec.lib()
    _set(L, jit_min_bytes=0)
    try:
        yield L
    finally:
        _set(L, jit=1, jit_min_bytes=64 << 20)


@pytest.fixture
def no_jit(swec):
    _set(swec.lib(), jit=0)
    try:
        yield
    finally:
        _set(swec.lib(), jit=1)


# ---------------------------------------------------------------------------------------------- helpers


def random_set(k, m, length, seed):
    rng = np.random.default_rng(seed)
    data = [rng.integers(0, 256, length, dtype=np.uint8) for _ in range(k)]
    return data + rn.encode(k, m, data)


def mask(n, lost):
    return tuple(i not in lost for i in range(n))


def write_set(base, shards, lost=()):
    for i, s in enumerate(shards):
        if i not in lost:
            s.tofile(base + ".ec%02d" % i)


def shard_paths(base, n=14):
    return [base + ".ec%02d" % i for i in range(n)]


def file_shards(base, ids):
    return {i: np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) for i in ids}


def snapshot(paths):
    return {p: (open(p, "rb").read(), os.stat(p).st_mtime_ns) for p in paths}


def age(paths):
    for p in paths:
        os.utime(p, ns=(PAST_NS, PAST_NS))


UNCHECKED = {"columns": 0, "damaged_columns": 0, "uncorrectable_columns": 0, "first_uncorrectable": -1,
             "last_uncorrectable": -1, "shards": {}, "ranges": [], "n_ranges": 0}


def heal_oracle(shards, k, m, present, radius):
    """(every shard after the heal: present ones corrected, lost ones rebuilt; report without "ok")."""
    present = tuple(bool(p) for p in present)
    info, checks, lost, _, r = do.punctured_rows(k, m, present)
    out = [s.copy() if present[i] else None for i, s in enumerate(shards)]
    c = len(checks)
    if c == 0:
        rep = dict(UNCHECKED)
    else:
        cols, a, b, va, vb, ids = do.decode_columns(shards, k, m, min(radius, c // 2), present)
        for pa, ev in ((a, va), (b, vb)):
            for p in np.unique(pa[pa >= 0]):
                sel = pa == p
                out[int(ids[p])][cols[sel]] ^= ev[sel]
        ida = np.where(a >= 0, ids[np.maximum(a, 0)], -1)
        idb = np.where(b >= 0, ids[np.maximum(b, 0)], -1)
        rep = do.report(len(shards[info[0]]), k + m, cols, ida, idb)
        del rep["ok"]
    for i, v in zip(lost, rn.apply_rows(r, [out[i] for i in info])):
        out[i] = v
    return out, rep


def damage_columns(shards, present, length, c, t, rng, extra=40):
    """Damage at every seam of the locate kernel, each column with a number of wrong present shards taken in turn from
    within t, t+1 .. c-t, and beyond c-t.  Returns {column: wrong shard count}."""
    ids = [i for i in range(len(shards)) if present[i]]
    seams = {0, 15, 16, 31, 32, 511, 512, 513, 4095, 4096, 4097, 8191, 8192, length // 16 * 16 - 1,
             length // 16 * 16, length - 1}
    cols = sorted(x for x in seams | set(rng.choice(length, size=extra, replace=False).tolist()) if 0 <= x < length)
    kinds = [w for w in (range(1, t + 1), range(t + 1, c - t + 1), range(c - t + 1, min(c + 2, len(ids)) + 1)) if len(w)]
    wrong = {}
    for n, col in enumerate(cols):
        kind = kinds[n % len(kinds)]
        w = int(kind[int(rng.integers(len(kind)))])
        for sid in rng.choice(ids, size=w, replace=False):
            shards[int(sid)][col] ^= np.uint8(rng.integers(1, 256))
        wrong[col] = w
    return wrong


# ------------------------------------------------------------------------------------------ CPU: argument rules


def _dev_args(L, enc, radius=1, report=True, ranges=True, cap=4, pres="ok", ptrs="ok"):
    from seaweedfs_b200._native import DamageRange, DamageReport
    rep, rng_arr, n = DamageReport(), (DamageRange * 4)(), C.c_int(0)
    present = {"ok": (C.c_uint8 * 14)(*([0] + [1] * 13)), "few": (C.c_uint8 * 14)(*([0] * 5 + [1] * 9)),
               None: None}[pres]
    p = {"ok": (C.c_void_p * 14)(*([1 << 20] * 14)), "lost_null": (C.c_void_p * 14)(*([None] + [1 << 20] * 13)),
         "present_null": (C.c_void_p * 14)(*([1 << 20] * 5 + [None] + [1 << 20] * 8)), None: None}[ptrs]
    return (enc, p, present, 4096, radius, C.byref(rep) if report else None, rng_arr if ranges else None, cap,
            C.byref(n), None)


DEVICE_CASES = [{"radius": -1}, {"radius": 3}, {"report": False}, {"cap": -1}, {"ranges": False}, {"pres": None},
                {"ptrs": None}, {"ptrs": "lost_null"}, {"ptrs": "present_null"}, {"pres": "few"},
                {"radius": 3, "report": False}, {"cap": -1, "ptrs": None}, {"pres": "few", "radius": 3},
                {"ptrs": "present_null", "pres": "few"}, {"ptrs": "lost_null", "cap": -1}, {"ranges": False, "cap": 0},
                {"radius": 0}, {"radius": 2}, {}]


def test_device_argument_rules_are_the_checked_reconstructs(swec):
    ec = swec.erasure_coding
    L = swec.lib()
    enc = ec.Encoder(10, 4, device=-1)
    for kw in DEVICE_CASES:
        got = (L.swec_heal_device(*_dev_args(L, enc._h, **kw)), L.swec_last_error())
        want = (L.swec_reconstruct_checked_device(*_dev_args(L, enc._h, **kw)), L.swec_last_error())
        assert got == want, kw
    assert L.swec_heal_device(*_dev_args(L, enc._h)) == -7           # SWEC_ERR_NO_DEVICE
    assert L.swec_heal_device(*_dev_args(L, None)) == -1
    with pytest.raises(swec.SwecError) as e:
        enc.heal_device([1 << 20] * 14, [0] + [1] * 13, 4096)
    assert e.value.name == "SWEC_ERR_NO_DEVICE"


def _file_call(L, fn, base, dirs=None, ndirs=0, k=10, m=4, device=-1, radius=1, report=True, cap=4, ranges=True,
               ok=True, rebuilt=True, n_rebuilt=True):
    from seaweedfs_b200._native import DamageRange, DamageReport
    rep, rng_arr, n, okv = DamageReport(), (DamageRange * 4)(), C.c_int(0), C.c_int(0)
    ids, n_ids = (C.c_uint32 * 32)(), C.c_int(7)
    rc = fn(base.encode() if base else None, dirs, ndirs, k, m, device, radius, ids if rebuilt else None,
            C.byref(n_ids) if n_rebuilt else None, C.byref(rep) if report else None, rng_arr if ranges else None, cap,
            C.byref(n), C.byref(okv) if ok else None)
    return rc, L.swec_last_error(), n_ids.value, okv.value


FILE_CASES = [{"radius": -1}, {"radius": 3}, {"report": False}, {"cap": -1}, {"ranges": False}, {"ok": False},
              {"rebuilt": False}, {"n_rebuilt": False}, {"base": None}, {"ndirs": 1},
              {"radius": 3, "report": False}, {"cap": -1, "ok": False}, {"base": None, "radius": 9},
              {"ranges": False, "cap": 0}, {"radius": 0}, {"radius": 2}, {"device": -1}, {"k": 6, "m": 3}, {}]


def test_file_argument_rules_are_the_checked_rebuilds(swec, tmp_path):
    L = swec.lib()
    base = str(tmp_path / "6")
    shards = random_set(10, 4, 100, 2)
    write_set(base, shards, lost=(0,))
    present = shard_paths(base)[1:]
    age(present)
    before = snapshot(present)
    for kw in FILE_CASES:
        kw = dict(kw)
        b = kw.pop("base", base)
        got = _file_call(L, L.swec_heal_ec_files, b, **kw)
        want = _file_call(L, L.swec_rebuild_ec_files_checked, b, **kw)
        assert got == want, kw
        assert not os.path.exists(base + ".ec00"), kw
    assert _file_call(L, L.swec_heal_ec_files, base)[:3] == (-7, L.swec_last_error(), 0)
    assert snapshot(present) == before
    # too few shards: the checked rebuild's error and text, before any output file exists
    for i in (1, 2, 3, 4):
        os.remove(base + ".ec%02d" % i)
    got = _file_call(L, L.swec_heal_ec_files, base)
    assert got == _file_call(L, L.swec_rebuild_ec_files_checked, base) and got[0] == -2
    assert b"found 9 shards, need at least 10" in got[1] and got[2] == 0
    assert sorted(os.listdir(tmp_path)) == sorted("6.ec%02d" % i for i in range(5, 14))
    # unequal lengths: the outputs are created, then removed
    shards[1][:50].tofile(base + ".ec01")
    for i in (2, 3, 4):
        shards[i].tofile(base + ".ec%02d" % i)
    got = _file_call(L, L.swec_heal_ec_files, base)
    assert got == _file_call(L, L.swec_rebuild_ec_files_checked, base) and got[0] == -6
    assert not os.path.exists(base + ".ec00")


def _volume_call(L, fn, base, index="", n_dirs=0, device=-1, rebuilt=True, n_rebuilt=True, heal=None):
    ids, n_ids = (C.c_uint32 * 32)(), C.c_int(7)
    args = [base.encode() if base else None, index.encode(), None, n_dirs, device, ids if rebuilt else None,
            C.byref(n_ids) if n_rebuilt else None]
    if heal is not None:
        from seaweedfs_b200._native import DamageRange, DamageReport
        rep, rng_arr, n, okv = DamageReport(), (DamageRange * 4)(), C.c_int(0), C.c_int(0)
        radius, report, ok = heal
        args[5:5] = [radius]
        args += [C.byref(rep) if report else None, rng_arr, 4, C.byref(n), C.byref(okv) if ok else None]
    rc = fn(*args)
    return rc, L.swec_last_error(), n_ids.value


def test_volume_argument_rules(swec, oracle, tmp_path):
    L = swec.lib()
    dat, idx = needle_volume(seed=5, needles=20)
    base, _ = lay_down(oracle, tmp_path, dat, idx)
    heal = (1, True, True)
    for kw in ({"base": None}, {"rebuilt": False}, {"n_rebuilt": False}, {"n_dirs": 1}):
        kw = dict(kw)
        b = kw.pop("base", base)
        got = _volume_call(L, L.swec_ec_shards_heal, b, heal=heal, **kw)
        assert got == _volume_call(L, L.swec_ec_shards_rebuild, b, **kw) and got[0] == -1, kw
    # nothing missing: the heal still checks the set, so it needs the device the plain rebuild does not
    assert _volume_call(L, L.swec_ec_shards_heal, base, heal=heal)[0] == -7
    # the heal's own rules are those of swec_heal_ec_files, which checks before any file is touched
    for radius, report, ok in ((3, True, True), (-1, True, True), (1, False, True), (1, True, False)):
        got = _volume_call(L, L.swec_ec_shards_heal, base, heal=(radius, report, ok))
        want = _file_call(L, L.swec_heal_ec_files, base, k=0, m=0, radius=radius, report=report, ok=ok)
        assert got[:2] == want[:2] and got[0] == -1, (radius, report, ok)
    # too few shards: swec_ec_shards_rebuild's error and text, nothing created, .ecx untouched
    ecx = open(base + ".ecx", "rb").read()
    for i in range(5):
        os.remove(base + ".ec%02d" % i)
    got = _volume_call(L, L.swec_ec_shards_heal, base, heal=heal)
    assert got == _volume_call(L, L.swec_ec_shards_rebuild, base) and got[0] == -2
    assert not any(os.path.exists(base + ".ec%02d" % i) for i in range(5))
    assert open(base + ".ecx", "rb").read() == ecx
    # a device-less call with shards to rebuild fails before the .ecx fold and leaves no output
    shards = oracle.encode_dat_image(dat, k=10, m=4)
    for i in range(1, 5):
        shards[i].tofile(base + ".ec%02d" % i)
    got = _volume_call(L, L.swec_ec_shards_heal, base, heal=heal)
    assert got == _volume_call(L, L.swec_ec_shards_rebuild, base) and got[0] == -7
    assert not os.path.exists(base + ".ec00")


# ------------------------------------------------------------------------------------------ GPU: device level


def _upload(torch, shards, present, length, shift):
    bufs = [torch.zeros(length + 32, dtype=torch.uint8, device="cuda") for _ in shards]
    for i, b in enumerate(bufs):
        if present[i]:
            b[shift:shift + length] = torch.from_numpy(shards[i]).cuda()
    return bufs


def _back(bufs, length, shift):
    return [b[shift:shift + length].cpu().numpy() for b in bufs]


DEVICE_GRID = [(10, 4, f, r) for f in range(5) for r in (0, 1, 2)] + \
              [(6, 3, f, r) for f in range(4) for r in (0, 1, 2)] + \
              [(12, 8, f, r) for f in range(9) for r in (0, 1)] + [(12, 8, 0, 2), (12, 8, 4, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", [(10, 4), (6, 3), (12, 8)])
def test_device_heal_against_the_oracle(cuda, swec, k, m):
    torch = cuda
    ec = swec.erasure_coding
    enc = ec.Encoder(k, m, device=0)
    length = 5 * 4096 + 13                   # a partial last vector
    for kk, mm, f, radius in DEVICE_GRID:
        if (kk, mm) != (k, m):
            continue
        rng = np.random.default_rng(k * 1000 + m * 100 + f * 10 + radius)
        clean = random_set(k, m, length, int(rng.integers(1 << 30)))
        lost = tuple(sorted(rng.choice(k + m, size=f, replace=False).tolist()))
        present = mask(k + m, lost)
        c = m - f
        t = min(radius, c // 2)
        shards = [s.copy() for s in clean]
        wrong = damage_columns(shards, present, length, c, t, rng)
        want, wrep = heal_oracle(shards, k, m, present, radius)
        for shift in (0, 3):                 # the vector path and the unaligned byte path
            what = (k, m, lost, radius, shift)
            hb = _upload(torch, shards, present, length, shift)
            rb = _upload(torch, shards, present, length, shift)
            got = enc.heal_device([b.data_ptr() + shift for b in hb], present, length, radius=radius)
            ref = enc.reconstruct_checked_device([b.data_ptr() + shift for b in rb], present, length, radius=radius)
            assert got == ref == wrep, what
            healed, checked = _back(hb, length, shift), _back(rb, length, shift)
            for i in range(k + m):
                assert (healed[i] == want[i]).all(), (what, i)
                if not present[i]:
                    assert (healed[i] == checked[i]).all(), (what, i)        # rebuilt: the checked rebuild's bytes
                assert (hb[i][:shift] == 0).all() and (hb[i][shift + length:] == 0).all(), (what, i)
            for col, w in wrong.items():
                if w <= t:                   # within t: the whole column is the true codeword
                    assert all(healed[i][col] == clean[i][col] for i in range(k + m)), (what, col)
                elif w <= c - t:             # reported: present bytes as found
                    assert rep_has_uncorrectable(got, col), (what, col)
                    assert all(healed[i][col] == shards[i][col] for i in range(k + m) if present[i]), (what, col)
            if f == 0 and radius >= 1 and 2 * radius <= m:
                cb = _upload(torch, shards, present, length, shift)
                cor = enc.correct_damage_device([b.data_ptr() + shift for b in cb], length, radius=radius)
                assert cor == got, what
                assert all((x == y).all() for x, y in zip(_back(cb, length, shift), healed)), what
            del hb, rb


def rep_has_uncorrectable(rep, col):
    return any(sid == -1 and off <= col < off + n for sid, off, n in rep["ranges"])


@pytest.mark.gpu
def test_device_heal_across_two_pieces(cuda, swec):
    """256 MiB + 4109 bytes per shard: the heal's second piece starts at 256 MiB.  Damage within the radius on both
    sides of the seam heals to the clean set; an uncorrectable column at the seam keeps its present bytes."""
    torch = cuda
    ec = swec.erasure_coding
    k, m = 10, 4
    n = (256 << 20) + 4109
    torch.manual_seed(7)
    clean = [torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda") for _ in range(k)]
    clean += [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(m)]
    enc = ec.Encoder(k, m, device=0)
    enc.encode_device([s.data_ptr() for s in clean[:k]], [s.data_ptr() for s in clean[k:]], n)
    enc.synchronize()
    present = mask(k + m, (6,))
    seam = 256 << 20
    shards = [s.clone() for s in clean]
    singles = {seam - 1: 2, seam: 11, seam + 16: 0, 5: 13, n - 1: 9, seam - 4096: 3}
    for col, sid in singles.items():
        shards[sid][col] ^= 0x5A
    shards[1][seam + 1] ^= 0x21                          # two wrong present shards: c = 3, t = 1, reported
    shards[12][seam + 1] ^= 0x84
    found = [s.clone() for s in shards]
    shards[6].zero_()
    checked = [s.clone() for s in shards]
    rep = enc.heal_device([s.data_ptr() for s in shards], present, n)
    ref = enc.reconstruct_checked_device([s.data_ptr() for s in checked], present, n)
    torch.cuda.synchronize()
    assert rep == ref
    assert rep["damaged_columns"] == len(singles) + 1 and rep["uncorrectable_columns"] == 1
    assert rep["first_uncorrectable"] == seam + 1
    assert rep["shards"] == {sid: (1, col, col) for col, sid in singles.items()}
    assert torch.equal(shards[6], checked[6])
    for i in range(k + m):
        d = (shards[i] != clean[i]).nonzero().flatten().tolist()
        if i in (1, 12):
            assert d == [seam + 1] and shards[i][seam + 1] == found[i][seam + 1], i
        elif i == 6:
            assert d in ([], [seam + 1]), d                 # rebuilt: plain rebuild's byte where uncorrectable
        else:
            assert d == [], (i, d)
    del shards, checked, found, clean
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ GPU: file level


def _copy(src_dir, dst_dir):
    shutil.copytree(src_dir, dst_dir)
    return dst_dir


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,lost,radius", [(10, 4, (5,), 1), (10, 4, (0, 13), 1), (10, 4, (), 2), (6, 3, (2,), 1),
                                             (10, 4, (3,), 0)])
def test_file_heal_against_the_oracle_and_the_two_call_flow(cuda, swec, tmp_path, no_jit, k, m, lost, radius):
    ec = swec.erasure_coding
    ctx = ec.ECContext(k, m)
    length = 3 * MIB
    rng = np.random.default_rng(k * 100 + len(lost) * 10 + radius)
    clean = random_set(k, m, length, int(rng.integers(1 << 30)))
    shards = [s.copy() for s in clean]
    present = mask(k + m, lost)
    ids = [i for i in range(k + m) if present[i]]
    cols = rng.choice(length, size=30 * len(ids[::3]), replace=False).reshape(-1, 30)
    for sid, sc in zip(ids[::3], cols):                  # scattered single-shard damage in a third of the shards
        shards[sid][sc] ^= rng.integers(1, 256, size=30, dtype=np.uint8)
    blamed_none = [i for i in ids if i not in ids[::3]]
    want, wrep = heal_oracle(shards, k, m, present, radius)
    src = tmp_path / "src"
    src.mkdir()
    write_set(str(src / "9"), shards, lost)
    age([shard_paths(str(src / "9"), k + m)[i] for i in ids])
    heal_dir, two_dir = _copy(src, tmp_path / "heal"), _copy(src, tmp_path / "two")
    hb, tb = str(heal_dir / "9"), str(two_dir / "9")
    untouched = [shard_paths(hb, k + m)[i] for i in blamed_none]
    before = snapshot(untouched)
    rep = ec.heal_ec_files(hb, ctx=ctx, radius=radius)
    chk = ec.rebuild_ec_files_checked(tb, ctx=ctx, radius=radius)
    assert rep == chk == {"rebuilt": list(lost), "ok": wrep["uncorrectable_columns"] == 0 and m - len(lost) >= 1, **wrep}
    healed = file_shards(hb, range(k + m))
    assert all((healed[i] == want[i]).all() for i in range(k + m))
    assert all((healed[i] == np.fromfile(tb + ".ec%02d" % i, dtype=np.uint8)).all() for i in lost)
    assert snapshot(untouched) == before                 # not blamed: neither written nor opened for writing
    if radius:
        assert all((healed[i] == clean[i]).all() for i in range(k + m))
        ec.repair_ec_damage(tb, ctx=ctx, radius=1)       # the completed set is within the repair's radius
        assert all((healed[i] == np.fromfile(tb + ".ec%02d" % i, dtype=np.uint8)).all() for i in range(k + m))
        again = ec.heal_ec_files(hb, ctx=ctx, radius=radius)
        assert again["damaged_columns"] == 0 and again["rebuilt"] == [] and again["ok"]
    else:
        assert all((healed[i] == shards[i]).all() for i in ids)          # radius 0 corrects nothing


def _miscorrectable_column():
    """RS(10,4) with shard 2 lost (c = 3, t = 1): errors e1, e4 in information shards 1 and 4 that, with the rebuilt
    byte of shard 2 they cause, make the completed column lie at distance 2 from another codeword c'.  c' is the
    weight-5 codeword on shards {1, 2, 4, 11, 13}: its data part x is zero but at 1, 2, 4 with x4 = 1, and parity rows 0
    and 2 vanish on it.  Returns (e1, e4, c') with c' a 14-vector."""
    g = rn.build_matrix(10, 14)
    p = g[10:]
    a = np.array([[p[0, 1], p[0, 2]], [p[2, 1], p[2, 2]]], dtype=np.uint8)
    rhs = np.array([p[0, 4], p[2, 4]], dtype=np.uint8)
    x12 = rn.mat_mul(rn.mat_inv(a), rhs[:, None])[:, 0]
    x = np.zeros(10, dtype=np.uint8)
    x[1], x[2], x[4] = x12[0], x12[1], 1
    cw = rn.mat_mul(g, x[:, None])[:, 0]
    assert sorted(np.flatnonzero(cw).tolist()) == [1, 2, 4, 11, 13]
    return int(cw[1]), int(cw[4]), cw


@pytest.mark.gpu
def test_heal_leaves_the_column_the_two_call_flow_miscorrects(cuda, swec, tmp_path, no_jit):
    ec = swec.erasure_coding
    length = MIB
    col = 123_457
    clean = random_set(10, 4, length, 77)
    shards = [s.copy() for s in clean]
    e1, e4, cw = _miscorrectable_column()
    shards[1][col] ^= np.uint8(e1)
    shards[4][col] ^= np.uint8(e4)
    src = tmp_path / "src"
    src.mkdir()
    write_set(str(src / "4"), shards, lost=(2,))
    hb, tb = str(_copy(src, tmp_path / "heal") / "4"), str(_copy(src, tmp_path / "two") / "4")
    present = [p for i, p in enumerate(shard_paths(hb)) if i != 2]
    age(present)
    before = snapshot(present)
    rep = ec.heal_ec_files(hb)
    assert rep["rebuilt"] == [2] and not rep["ok"] and rep["shards"] == {}
    assert rep["uncorrectable_columns"] == 1 and rep["first_uncorrectable"] == col
    assert snapshot(present) == before                   # present shards as found
    plain = do.punctured_rows(10, 4, mask(14, (2,)))
    rebuilt = rn.apply_rows(plain[4], [shards[i] for i in plain[0]])[0]
    assert (np.fromfile(hb + ".ec02", dtype=np.uint8) == rebuilt).all()
    # the two-call flow: the checked rebuild, then the repair at radius 2 on the completed set
    assert ec.rebuild_ec_files_checked(tb)["uncorrectable_columns"] == 1
    rep2 = ec.repair_ec_damage(tb, radius=2)
    assert set(rep2["shards"]) == {11, 13} and rep2["uncorrectable_columns"] == 0
    two = file_shards(tb, range(14))
    column = np.array([two[i][col] for i in range(14)], dtype=np.uint8)
    assert (column == (np.array([clean[i][col] for i in range(14)], dtype=np.uint8) ^ cw)).all()   # another codeword


@pytest.mark.gpu
def test_clean_set_is_not_written_and_pass_2_reads_only_flagged_pages(cuda, swec, tmp_path, no_jit, capfd,
                                                                      monkeypatch):
    ec = swec.erasure_coding
    length = 8 * MIB
    clean = random_set(10, 4, length, 88)
    base = str(tmp_path / "5")
    write_set(base, clean, lost=(12,))
    present = [p for i, p in enumerate(shard_paths(base)) if i != 12]
    age(present)
    before = snapshot(present)
    monkeypatch.setenv("SWEC_PIPE_STATS", "1")
    capfd.readouterr()
    rep = ec.heal_ec_files(base)
    assert rep["ok"] and rep["damaged_columns"] == 0 and rep["rebuilt"] == [12]
    assert snapshot(present) == before
    assert (np.fromfile(base + ".ec12", dtype=np.uint8) == clean[12]).all()
    pipes = [json.loads(x) for x in capfd.readouterr().err.splitlines() if x.startswith('{"pipe"')]
    assert [p["pipe"] for p in pipes] == ["heal_ec_files"]
    # damage in three pages of one shard, one of them also uncorrectable: pass 2 reads only their page spans
    os.remove(base + ".ec12")
    for col in (5 * 4096 + 7, 5 * 4096 + 9, 700 * 4096, 1500 * 4096 + 4095):
        flip(base + ".ec03", col)
    flip(base + ".ec08", 1500 * 4096 + 4095)
    capfd.readouterr()
    rep = ec.heal_ec_files(base)
    assert rep["shards"] == {3: (3, 5 * 4096 + 7, 700 * 4096)} and rep["uncorrectable_columns"] == 1
    pipes = {p["pipe"]: p for p in (json.loads(x) for x in capfd.readouterr().err.splitlines()
                                    if x.startswith('{"pipe"'))}
    assert set(pipes) == {"heal_ec_files", "heal_pages"}
    assert pipes["heal_pages"]["items"] <= 3              # one item per flagged page at most


def flip(path, off, mask=0x40):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ mask]))


@pytest.mark.gpu
def test_failure_leaves_no_rebuilt_file_and_no_ids(cuda, swec, tmp_path, no_jit):
    """A length above 1 MiB that is not a whole number of MiB fails after pass 1 ran (the rebuild's quirk): no rebuilt
    file is left, no id is reported and pass 2 does not run."""
    L = swec.lib()
    length = MIB + 4096
    shards = random_set(10, 4, length, 99)
    shards[0][100] ^= 1
    base = str(tmp_path / "r")
    write_set(base, shards, lost=(7,))
    present = [p for i, p in enumerate(shard_paths(base)) if i != 7]
    age(present)
    before = snapshot(present)
    got = _file_call(L, L.swec_heal_ec_files, base, device=0)
    assert got[0] == -6 and got[2] == 0 and got[3] == 0
    assert not os.path.exists(base + ".ec07") and snapshot(present) == before


@pytest.mark.gpu
def test_volume_heal_folds_the_ecj(cuda, swec, oracle, tmp_path, no_jit):
    ec = swec.erasure_coding
    dat, idx = needle_volume(seed=21, needles=150)
    (tmp_path / "h").mkdir()
    (tmp_path / "r").mkdir()
    bases = {}
    for name in ("h", "r"):
        base, clean = lay_down(oracle, tmp_path / name, dat, idx)
        keys = [k for k, _, _ in rn._entries(rn.sorted_ecx_from_idx(idx))]
        open(base + ".ecj", "wb").write(b"".join(k.to_bytes(8, "big") for k in keys[:2]))
        os.remove(base + ".ec11")
        flip(base + ".ec02", len(clean[2]) // 2)
        bases[name] = base
    rep = ec.volume_ec_shards_heal(bases["h"])
    assert rep["rebuilt"] == [11] and rep["ok"] and rep["shards"] == {2: (1, len(clean[2]) // 2, len(clean[2]) // 2)}
    assert ec.volume_ec_shards_rebuild(bases["r"]) == [11]
    for name in ("h", "r"):
        assert not os.path.exists(bases[name] + ".ecj")
    assert open(bases["h"] + ".ecx", "rb").read() == open(bases["r"] + ".ecx", "rb").read()
    assert all((np.fromfile(bases["h"] + ".ec%02d" % i, dtype=np.uint8) == clean[i]).all() for i in range(14))
