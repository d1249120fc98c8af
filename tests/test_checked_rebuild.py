"""The checked rebuild: swec_rebuild_ec_files_checked (shard files) and swec_reconstruct_checked_device (shards in HBM),
errors and erasures on the punctured code, checked against an oracle that shares nothing with the kernel's method.

The oracle takes the first k present shards as the information set I and the other c present shards as the check set C,
builds P' = G[C]·G[I]^-1 and R = G[lost]·G[I]^-1 from oracle.rs_numpy (build_matrix, mat_inv), and decodes every column
by exhaustive lookup over every pattern of up to t = min(radius, c // 2) wrong present shards with every error value,
as tests/damage_oracle.py does for the full code.  Located errors in I are corrected before R rebuilds the lost shards;
other columns are rebuilt from I as found.

cpu: every 1x1 and 2x2 minor of P' is non-zero for every presence pattern of RS(10,4); the oracle restores up to t
errors plus f erasures and reports t+1 .. c-t; the argument rules of both calls, each failing before any file exists;
no device; too few shards and unequal lengths with the texts of swec_rebuild_ec_files.
gpu: clean sets with 1-4 lost shards (files equal plain rebuild's and the originals, present files untouched); one lost
shard plus one flipped byte in each present shard (then repair restores all 14 files); scattered damage with 1 and 2
lost; two wrong shards in a column; radius 0 with 3 lost; nothing lost; radius 2 on RS(8,6); slot boundary, long run and
tail; an additional directory; O_DIRECT; fuzz at file and device level; 13 x 3 GiB in HBM."""
import ctypes as C
import functools
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import damage_oracle as do  # noqa: E402

from oracle import rs_numpy as rn  # noqa: E402

SEED = 0x5EC7
GIB = 1 << 30
PAST_NS = 1_000_000_000 * 1_000_000_000    # an mtime no write can produce


# ---------------------------------------------------------------------------------------------- helpers


def random_set(k, m, length, seed):
    rng = np.random.default_rng(seed)
    data = [rng.integers(0, 256, length, dtype=np.uint8) for _ in range(k)]
    return data + rn.encode(k, m, data)


def write_set(base, shards, lost=()):
    for i, s in enumerate(shards):
        if i not in lost:
            s.tofile(base + ".ec%02d" % i)


def file_shards(base, n=14):
    return [np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) for i in range(n)]


def shard_paths(base, n=14):
    return [base + ".ec%02d" % i for i in range(n)]


def same(a, b):
    return len(a) == len(b) and all((x == y).all() for x, y in zip(a, b))


def age(paths):
    for p in paths:
        os.utime(p, ns=(PAST_NS, PAST_NS))


def snapshot(paths):
    return {p: (open(p, "rb").read(), os.stat(p).st_mtime_ns) for p in paths}


def flip(path, off, mask=0x40):
    with open(path, "r+b") as f:
        f.seek(off)
        b = f.read(1)
        f.seek(off)
        f.write(bytes([b[0] ^ mask]))


def damage(shards, columns, rng, choose):
    for c in columns:
        for sid in choose:
            shards[int(sid)][c] ^= np.uint8(rng.integers(1, 256))


# ---------------------------------------------------------------------------------------------- errors-and-erasures oracle


def punctured(k, m, present):
    """(info ids, check ids, lost ids, P' c x k, R f x k) for a presence mask."""
    g = rn.build_matrix(k, k + m)
    ids = [i for i in range(k + m) if present[i]]
    info = ids[:k]
    checks = ids[k:]
    lost = [i for i in range(k + m) if not present[i]]
    ginv = rn.mat_inv(g[info])
    pc = rn.mat_mul(g[checks], ginv) if checks else np.zeros((0, k), dtype=np.uint8)
    r = rn.mat_mul(g[lost], ginv) if lost else np.zeros((0, k), dtype=np.uint8)
    return info, checks, lost, pc, r


@functools.lru_cache(maxsize=None)
def _table(k, m, present, t):
    """Sorted syndrome keys of every pattern of 1..t wrong positions of the punctured code (positions: k information,
    then c check), with positions a, b (-1: none) and error values va, vb."""
    _, _, _, pc, _ = punctured(k, m, present)
    c = pc.shape[0]
    h = np.concatenate([pc, np.eye(c, dtype=np.uint8)], axis=1)
    n = k + c
    e = np.arange(1, 256, dtype=np.uint8)
    cols = [rn.MUL[e[:, None], h[:, j][None, :]] for j in range(n)]
    keys, a, b, va, vb = [], [], [], [], []
    if t >= 1:
        for j in range(n):
            keys.append(do._keys(cols[j]))
            a.append(np.full(255, j, dtype=np.int16))
            b.append(np.full(255, -1, dtype=np.int16))
            va.append(e)
            vb.append(np.zeros(255, dtype=np.uint8))
    if t >= 2:
        for x in range(n):
            for y in range(x + 1, n):
                keys.append(do._keys(cols[x][:, None, :] ^ cols[y][None, :, :]).ravel())
                a.append(np.full(255 * 255, x, dtype=np.int16))
                b.append(np.full(255 * 255, y, dtype=np.int16))
                va.append(np.repeat(e, 255))
                vb.append(np.tile(e, 255))
    if not keys:
        z = np.zeros(0, dtype=np.uint64)
        return z, z.astype(np.int16), z.astype(np.int16), z.astype(np.uint8), z.astype(np.uint8)
    keys, a, b, va, vb = (np.concatenate(v) for v in (keys, a, b, va, vb))
    order = np.argsort(keys, kind="stable")
    keys = keys[order]
    assert (np.diff(keys) != 0).all(), "two patterns within the radius share a syndrome: the punctured code is not MDS"
    return keys, a[order], b[order], va[order], vb[order]


def checked_rebuild(shards, k, m, present, radius=1):
    """What the checked rebuild gives for the shards (lost ones may be None): ({lost id: rebuilt bytes}, report)."""
    present = tuple(bool(p) for p in present)
    info, checks, lost, pc, r = punctured(k, m, present)
    length = len(shards[info[0]])
    x = [shards[i].copy() for i in info]
    c = len(checks)
    if c == 0:
        rep = {"ok": False, "columns": 0, "damaged_columns": 0, "uncorrectable_columns": 0, "first_uncorrectable": -1,
               "last_uncorrectable": -1, "shards": {}, "ranges": [], "n_ranges": 0}
        return dict(zip(lost, rn.apply_rows(r, x))), rep
    t = min(radius, c // 2)
    comp = rn.apply_rows(pc, x)
    s = np.stack([comp[i] ^ shards[checks[i]] for i in range(c)], axis=1)
    cols = np.flatnonzero(s.any(axis=1))
    keys, a, b, va, vb = _table(k, m, present, t)
    if len(keys):
        q = do._keys(s[cols])
        pos = np.minimum(np.searchsorted(keys, q), len(keys) - 1)
        found = keys[pos] == q
    else:
        pos, found = np.zeros(len(cols), dtype=np.int64), np.zeros(len(cols), dtype=bool)
    ca, cb = (np.where(found, w[pos] if len(w) else -1, -1) for w in (a, b))
    ea, eb = (np.where(found, v[pos] if len(v) else 0, 0).astype(np.uint8) for v in (va, vb))
    for pa, ev in ((ca, ea), (cb, eb)):                  # errors of information positions come out before R
        for j in range(k):
            sel = pa == j
            x[j][cols[sel]] ^= ev[sel]
    ids = np.array(info + checks, dtype=np.int64)
    ida = np.where(ca >= 0, ids[np.maximum(ca, 0)], -1)
    idb = np.where(cb >= 0, ids[np.maximum(cb, 0)], -1)
    rep = do.report(length, k + m, cols, ida, idb)
    rep["ok"] = rep["uncorrectable_columns"] == 0
    return dict(zip(lost, rn.apply_rows(r, x))), rep


def plain_rebuild(shards, k, m, present):
    info, _, lost, _, r = punctured(k, m, tuple(bool(p) for p in present))
    return dict(zip(lost, rn.apply_rows(r, [shards[i] for i in info])))


def mask(n, lost):
    return tuple(i not in lost for i in range(n))


# ------------------------------------------------------------------------------------------ CPU


def test_every_small_minor_of_the_punctured_check_rows_is_non_zero():
    k, m = 10, 4
    patterns = 0
    for f in range(m + 1):
        for lost in itertools.combinations(range(k + m), f):
            _, _, _, pc, _ = punctured(k, m, mask(k + m, lost))
            patterns += 1
            assert (pc != 0).all(), lost
            for r0, r1 in itertools.combinations(range(pc.shape[0]), 2):
                det = rn.MUL[pc[r0][:, None], pc[r1][None, :]] ^ rn.MUL[pc[r0][None, :], pc[r1][:, None]]
                off = ~np.eye(k, dtype=bool)
                assert (det[off] != 0).all(), (lost, r0, r1)
    assert patterns == 1 + 14 + 91 + 364 + 1001


@pytest.mark.parametrize("k,m", [(10, 4), (8, 6), (6, 3)])
def test_oracle_corrects_errors_and_erasures(k, m):
    rng = np.random.default_rng(k * 100 + m)
    length = 2000
    for f in range(m):
        lost = tuple(sorted(rng.choice(k + m, size=f, replace=False).tolist()))
        present = mask(k + m, lost)
        _, checks, _, _, _ = punctured(k, m, present)
        c = len(checks)
        for radius in (0, 1, 2):
            t = min(radius, c // 2)
            for wrong in range(1, c - t + 1):
                clean = random_set(k, m, length, seed=f * 10 + wrong)
                shards = [s.copy() for s in clean]
                cols = np.sort(rng.choice(length, size=150, replace=False))
                ids = [i for i in range(k + m) if present[i]]
                for col in cols:
                    damage(shards, [col], rng, rng.choice(ids, size=wrong, replace=False))
                got, rep = checked_rebuild(shards, k, m, present, radius)
                assert rep["damaged_columns"] == len(cols)
                if wrong <= t:
                    assert all((got[i] == clean[i]).all() for i in lost), (lost, radius, wrong)
                    assert rep["uncorrectable_columns"] == 0 and rep["ok"]
                else:                   # t < wrong <= c - t: reported, and rebuilt as plain rebuild does
                    assert rep["uncorrectable_columns"] == len(cols) and not rep["ok"] and rep["shards"] == {}
                    plain = plain_rebuild(shards, k, m, present)
                    assert all((got[i] == plain[i]).all() for i in lost), (lost, radius, wrong)


def _call_file(L, base, radius=1, report=True, cap=4, ranges=True, ok=True, rebuilt=True, device=-1):
    from seaweedfs_b200._native import DamageRange, DamageReport
    rep, rng_arr, n, okv = DamageReport(), (DamageRange * 4)(), C.c_int(0), C.c_int(0)
    ids, n_ids = (C.c_uint32 * 32)(), C.c_int(7)
    rc = L.swec_rebuild_ec_files_checked(base.encode(), None, 0, 10, 4, device, radius, ids if rebuilt else None,
                                         C.byref(n_ids), C.byref(rep) if report else None, rng_arr if ranges else None,
                                         cap, C.byref(n), C.byref(okv) if ok else None)
    return rc, n_ids.value


def test_checked_argument_rules(swec, tmp_path):
    from seaweedfs_b200._native import DamageRange, DamageReport
    ec = swec.erasure_coding
    L = swec.lib()
    base = str(tmp_path / "6")
    shards = random_set(10, 4, 100, 2)
    write_set(base, shards, lost=(0,))
    age(shard_paths(base)[1:])
    before = snapshot(shard_paths(base)[1:])
    for kw in ({"radius": -1}, {"radius": 3}, {"report": False}, {"cap": -1}, {"ranges": False}, {"ok": False},
               {"rebuilt": False}):
        rc, n_ids = _call_file(L, base, **kw)
        assert rc == -1, kw
        assert n_ids == (7 if kw in ({"rebuilt": False}, {"ok": False}) else 0), kw   # NULL pointers: nothing written
        assert not os.path.exists(base + ".ec00"), kw
    assert _call_file(L, base, radius=3)[0] == -1 and b"radius must be 0, 1 or 2" in L.swec_last_error()
    for radius in (0, 1, 2):                               # valid: on to the device, whose absence removes the output
        assert _call_file(L, base, radius=radius) == (-7, 0)
        assert not os.path.exists(base + ".ec00")
    assert _call_file(L, base, ranges=False, cap=0) == (-7, 0)
    assert snapshot(shard_paths(base)[1:]) == before

    rep, rng_arr, n = DamageReport(), (DamageRange * 4)(), C.c_int(0)
    e104 = ec.Encoder(10, 4, device=-1)
    present = (C.c_uint8 * 14)(*([0] + [1] * 13))
    ptrs = (C.c_void_p * 14)(*([1 << 20] * 14))

    def dev_call(radius=1, report=C.byref(rep), ranges=rng_arr, cap=4, pres=present, p=ptrs):
        return L.swec_reconstruct_checked_device(e104._h, p, pres, 4096, radius, report, ranges, cap, C.byref(n), None)

    for kw in ({"radius": -1}, {"radius": 3}, {"report": None}, {"cap": -1}, {"ranges": None}, {"pres": None},
               {"p": None}):
        assert dev_call(**kw) == -1, kw
    assert dev_call(p=(C.c_void_p * 14)(*([None] + [1 << 20] * 13))) == -1     # the shard to rebuild has no buffer
    assert dev_call(p=(C.c_void_p * 14)(*([1 << 20] * 5 + [None] + [1 << 20] * 8))) == -1   # a present shard has none
    assert dev_call(pres=(C.c_uint8 * 14)(*([0] * 5 + [1] * 9))) == -2
    for radius in (0, 1, 2):
        assert dev_call(radius=radius) == -7
    assert dev_call(ranges=None, cap=0) == -7


def test_checked_without_a_device(swec, tmp_path):
    ec = swec.erasure_coding
    enc = ec.Encoder(10, 4, device=-1)
    with pytest.raises(swec.SwecError) as e:
        enc.reconstruct_checked_device([1 << 20] * 14, [0] + [1] * 13, 4096)
    assert e.value.name == "SWEC_ERR_NO_DEVICE"
    base = str(tmp_path / "5")
    write_set(base, random_set(10, 4, 5000, 1), lost=(3, 12))
    before = snapshot([p for p in shard_paths(base) if os.path.exists(p)])
    with pytest.raises(swec.SwecError) as e:
        ec.rebuild_ec_files_checked(base, device=-1)
    assert e.value.name == "SWEC_ERR_NO_DEVICE"
    assert sorted(os.listdir(tmp_path)) == sorted("5.ec%02d" % i for i in range(14) if i not in (3, 12))
    assert snapshot([p for p in shard_paths(base) if os.path.exists(p)]) == before
    L = swec.lib()
    assert _call_file(L, base) == (-7, 0)


def test_checked_file_checks_match_plain_rebuild(swec, tmp_path):
    ec = swec.erasure_coding
    base = str(tmp_path / "8")
    shards = random_set(10, 4, 1000, 3)
    write_set(base, shards, lost=(0, 4, 7, 9, 13))
    texts = []
    for call in (ec.rebuild_ec_files, ec.rebuild_ec_files_checked):
        with pytest.raises(swec.SwecError) as e:
            call(base, device=-1)
        assert e.value.name == "SWEC_ERR_TOO_FEW_SHARDS"
        texts.append(str(e.value))
    assert texts[0] == texts[1] and "found 9 shards, need at least 10" in texts[0]
    assert sorted(os.listdir(tmp_path)) == sorted("8.ec%02d" % i for i in range(14) if i not in (0, 4, 7, 9, 13))
    shards[0].tofile(base + ".ec00")
    with open(base + ".ec11", "ab") as f:
        f.write(b"x")
    texts = []
    for call in (ec.rebuild_ec_files, ec.rebuild_ec_files_checked):
        with pytest.raises(swec.SwecError) as e:
            call(base, device=-1)
        assert e.value.name == "SWEC_ERR_SHARD_SIZE"
        texts.append(str(e.value))
    assert texts[0] == texts[1] and texts[0].endswith("ec shard size expected 1000 actual 1001")
    for i in (4, 7, 9, 13):
        assert not os.path.exists(base + ".ec%02d" % i)
    # the outputs are created before the lengths are compared: an output that cannot be created fails first
    disk = tmp_path / "disk2"
    disk.mkdir()
    for i in range(14):
        if os.path.exists(base + ".ec%02d" % i):
            os.rename(base + ".ec%02d" % i, str(disk / ("8.ec%02d" % i)))
    gone = str(tmp_path / "gone" / "8")
    with pytest.raises(swec.SwecError) as e:
        ec.rebuild_ec_files_checked(gone, [str(disk)], device=-1)
    assert e.value.name == "SWEC_ERR_IO" and f"create {gone}.ec04: " in str(e.value)


# ------------------------------------------------------------------------------------------ GPU


def mtimes(paths):
    return [os.stat(p).st_mtime_ns for p in paths]


def run_checked(ec, base, lost, radius=1, **kw):
    """The checked rebuild on a set whose `lost` files were removed: (report, rebuilt shards by id)."""
    rep = ec.rebuild_ec_files_checked(base, radius=radius, **kw)
    assert rep["rebuilt"] == sorted(lost)
    got = {i: np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) for i in lost}
    return rep, got


def remove(base, lost):
    for i in lost:
        os.remove(base + ".ec%02d" % i)


@pytest.mark.gpu
def test_clean_set_every_loss_pattern(cuda, swec, oracle, tmp_path):
    ec = swec.erasure_coding
    size = 5_432_109
    base = str(tmp_path / "21")
    oracle.synth(0, size, SEED).tofile(base + ".dat")
    ec.write_ec_files(base)
    clean = file_shards(base)
    patterns = [(i,) for i in range(14)] + [(0, 13), (3, 9), (10, 11), (0, 5, 12), (1, 2, 3), (0, 1, 2, 3),
                                            (6, 10, 12, 13)]
    for lost in patterns:
        present_paths = [p for i, p in enumerate(shard_paths(base)) if i not in lost]
        remove(base, lost)
        plain = ec.rebuild_ec_files(base)
        assert plain == list(lost)
        plain_bytes = {i: np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) for i in lost}
        remove(base, lost)
        age(present_paths)
        before = snapshot(present_paths)
        rep, got = run_checked(ec, base, lost)
        c = 4 - len(lost)
        assert rep["ok"] == (c >= 1), lost
        assert rep["columns"] == (len(clean[0]) if c else 0) and rep["damaged_columns"] == 0 and rep["shards"] == {}
        for i in lost:
            assert (got[i] == clean[i]).all() and (got[i] == plain_bytes[i]).all(), (lost, i)
        assert snapshot(present_paths) == before, lost


@pytest.mark.gpu
def test_one_lost_one_flipped_byte_in_each_present_shard(cuda, swec, oracle, tmp_path):
    ec = swec.erasure_coding
    size = 9_876_543
    base = str(tmp_path / "22")
    oracle.synth(0, size, SEED + 1).tofile(base + ".dat")
    ec.write_ec_files(base)
    clean = file_shards(base)
    shard_len = len(clean[0])
    lost = 4
    for sid in [i for i in range(14) if i != lost]:
        write_set(base, clean, lost=(lost,))
        if os.path.exists(base + ".ec%02d" % lost):
            remove(base, (lost,))
        off = (654_321 * (sid + 1)) % shard_len
        flip(base + ".ec%02d" % sid, off)
        plain = ec.rebuild_ec_files(base)
        assert plain == [lost]
        wrong_plain = np.fromfile(base + ".ec%02d" % lost, dtype=np.uint8)
        first_k = [i for i in range(14) if i != lost][:10]
        assert (wrong_plain != clean[lost]).any() == (sid in first_k), sid
        remove(base, (lost,))
        rep, got = run_checked(ec, base, (lost,))
        assert rep["ok"] and rep["damaged_columns"] == 1 and rep["uncorrectable_columns"] == 0, sid
        assert rep["shards"] == {sid: (1, off, off)}, sid
        assert (got[lost] == clean[lost]).all(), sid
        rep2 = ec.repair_ec_damage(base)
        assert rep2["ok"] and rep2["shards"] == {sid: (1, off, off)}, sid
        assert same(file_shards(base), clean), sid


@pytest.mark.gpu
@pytest.mark.parametrize("lost", [(2,), (0, 11)])
def test_scattered_single_shard_damage(cuda, swec, tmp_path, lost):
    ec = swec.erasure_coding
    length = 777_777
    clean = random_set(10, 4, length, 31 + len(lost))
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(32)
    present_ids = [i for i in range(14) if i not in lost]
    for n, sid in enumerate(present_ids):
        cols = np.sort(rng.choice(4096, size=200, replace=False)) + (7 * n + 1) * 4096
        damage(shards, cols, rng, [sid])
    base = str(tmp_path / "s")
    write_set(base, shards, lost=lost)
    want, wrep = checked_rebuild(shards, 10, 4, mask(14, lost))
    assert wrep["uncorrectable_columns"] == 0 and len(wrep["shards"]) == 14 - len(lost)
    rep, got = run_checked(ec, base, lost)
    assert rep == {"rebuilt": list(lost), **wrep}
    for i in lost:
        assert (got[i] == want[i]).all() and (got[i] == clean[i]).all()


@pytest.mark.gpu
def test_two_wrong_present_shards_in_a_column(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    length = 300_000
    clean = random_set(10, 4, length, 41)
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(42)
    damage(shards, np.arange(10_000, 20_000), rng, [1])
    damage(shards, np.arange(15_000, 25_000), rng, [12])     # overlap 15,000..19,999
    base = str(tmp_path / "2w")
    write_set(base, shards, lost=(5,))
    want, wrep = checked_rebuild(shards, 10, 4, mask(14, (5,)))
    rep, got = run_checked(ec, base, (5,))
    assert rep == {"rebuilt": [5], **wrep} and not rep["ok"]
    assert rep["uncorrectable_columns"] == 5_000 and rep["first_uncorrectable"] == 15_000
    assert (got[5] == want[5]).all()
    plain = plain_rebuild(shards, 10, 4, mask(14, (5,)))[5]
    assert (got[5][15_000:20_000] == plain[15_000:20_000]).all()
    assert (got[5][:15_000] == clean[5][:15_000]).all() and (got[5][20_000:] == clean[5][20_000:]).all()


@pytest.mark.gpu
def test_three_lost_and_radius_0(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    length = 200_003
    clean = random_set(10, 4, length, 51)
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(52)
    damage(shards, np.arange(1000, 1100), rng, [3])
    damage(shards, np.arange(50_000, 50_010), rng, [13])
    damage(shards, [length - 1], rng, [7])
    for lost, radius in (((0, 1, 2), 1), ((0, 1, 2), 0), ((4, 10), 0), ((9,), 0)):
        base = str(tmp_path / ("r%d_%d" % (radius, len(lost))))
        write_set(base, shards, lost=lost)
        want, wrep = checked_rebuild(shards, 10, 4, mask(14, lost), radius)
        rep, got = run_checked(ec, base, lost, radius=radius)
        assert rep == {"rebuilt": list(lost), **wrep}, (lost, radius)
        assert rep["shards"] == {} and rep["uncorrectable_columns"] == 111 and not rep["ok"]
        plain = plain_rebuild(shards, 10, 4, mask(14, lost))
        for i in lost:
            assert (got[i] == plain[i]).all() and (got[i] == want[i]).all(), (lost, radius, i)


@pytest.mark.gpu
def test_nothing_lost_reports_what_locate_reports(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    length = 400_000
    shards = random_set(10, 4, length, 61)
    rng = np.random.default_rng(62)
    damage(shards, np.arange(100, 400), rng, [2])
    damage(shards, np.arange(300, 350), rng, [11])
    damage(shards, np.arange(90_000, 95_000), rng, [13])
    base = str(tmp_path / "n")
    write_set(base, shards)
    age(shard_paths(base))
    before = snapshot(shard_paths(base))
    for radius in (1, 2):
        loc = ec.locate_ec_damage(base, radius=radius)
        rep = ec.rebuild_ec_files_checked(base, radius=radius)
        assert rep["rebuilt"] == []
        assert {k: v for k, v in rep.items() if k not in ("ok", "rebuilt")} == \
            {k: v for k, v in loc.items() if k != "ok"}, radius
        assert rep["ok"] == (loc["uncorrectable_columns"] == 0)
    rep0 = ec.rebuild_ec_files_checked(base, radius=0)
    assert rep0["shards"] == {} and rep0["uncorrectable_columns"] == rep0["damaged_columns"] == 5_300
    assert snapshot(shard_paths(base)) == before


@pytest.mark.gpu
def test_radius_2_on_rs_8_6(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    k, m = 8, 6
    length = 250_000
    clean = random_set(k, m, length, 71)
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(72)
    damage(shards, np.arange(1000, 9000), rng, [0])
    damage(shards, np.arange(5000, 13_000), rng, [10])      # overlap: two wrong present shards, c = 5, t = 2
    damage(shards, np.arange(100_000, 100_100), rng, [4, 9, 12])    # three: reported
    base = str(tmp_path / "86")
    write_set(base, shards, lost=(3,))
    ctx = ec.ECContext(k, m)
    want, wrep = checked_rebuild(shards, k, m, mask(k + m, (3,)), 2)
    rep = ec.rebuild_ec_files_checked(base, ctx=ctx, radius=2)
    assert rep == {"rebuilt": [3], **wrep}
    assert rep["uncorrectable_columns"] == 100 and set(rep["shards"]) == {0, 10}
    got = np.fromfile(base + ".ec03", dtype=np.uint8)
    assert (got == want[3]).all()
    assert (got[:100_000] == clean[3][:100_000]).all() and (got[100_100:] == clean[3][100_100:]).all()


@pytest.mark.gpu
def test_slot_boundary_long_run_and_tail(cuda, swec, tmp_path, monkeypatch):
    ec = swec.erasure_coding
    monkeypatch.setenv("SWEC_FILE_CHUNK", str(64 << 10))
    length = 1_000_003
    clean = random_set(10, 4, length, 81)
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(82)
    first = 3 * (64 << 10) - 2000
    damage(shards, np.arange(first, first + 4096 + 77), rng, [3])
    damage(shards, np.arange(400_000, 550_000), rng, [11])
    damage(shards, np.arange(length - 1000, length), rng, [6])
    damage(shards, [length - 1], rng, [13])                   # the last column: two wrong shards
    base = str(tmp_path / "3")
    write_set(base, shards, lost=(1,))
    want, wrep = checked_rebuild(shards, 10, 4, mask(14, (1,)))
    rep, got = run_checked(ec, base, (1,))
    assert rep == {"rebuilt": [1], **wrep}
    assert rep["uncorrectable_columns"] == 1 and rep["first_uncorrectable"] == length - 1
    assert (got[1] == want[1]).all() and (got[1][:-1] == clean[1][:-1]).all()


@pytest.mark.gpu
def test_present_shard_in_an_additional_directory(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    length = 500_000
    clean = random_set(10, 4, length, 91)
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(92)
    damage(shards, np.arange(70_000, 80_000), rng, [9])
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    base, other = str(tmp_path / "a" / "7"), str(tmp_path / "b" / "7")
    for i, s in enumerate(shards):
        if i != 2:
            s.tofile((other if i >= 8 else base) + ".ec%02d" % i)
    rep = ec.rebuild_ec_files_checked(base, additional_dirs=[str(tmp_path / "b")])
    assert rep["rebuilt"] == [2] and rep["ok"] and rep["shards"] == {9: (10_000, 70_000, 79_999)}
    assert (np.fromfile(base + ".ec02", dtype=np.uint8) == clean[2]).all()


@pytest.mark.gpu
def test_checked_rebuild_with_o_direct(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    L = swec.lib()
    length = 3 * (8 << 20) + (1 << 20)     # a whole number of MiB: rebuild refuses other lengths above 1 MiB
    clean = random_set(10, 4, length, 101)
    shards = [s.copy() for s in clean]
    rng = np.random.default_rng(102)
    damage(shards, np.arange(8 << 20, (8 << 20) + 3 * 4096), rng, [0])
    damage(shards, np.arange(length - 200, length), rng, [6])
    base = str(tmp_path / "d")
    write_set(base, shards, lost=(12,))
    assert L.swec_set_option(b"file_direct_io", 3) == 0
    try:
        rep, got = run_checked(ec, base, (12,))
    finally:
        assert L.swec_set_option(b"file_direct_io", int(os.environ.get("SWEC_FILE_DIRECT", "0")) & 3) == 0
    want, wrep = checked_rebuild(shards, 10, 4, mask(14, (12,)))
    assert rep == {"rebuilt": [12], **wrep} and rep["ok"]
    assert (got[12] == clean[12]).all()


FUZZ = [(10, 4, (0,)), (10, 4, (3, 11)), (10, 4, ()), (6, 3, (8,)), (8, 6, (0, 1)), (12, 6, (5, 17)),
        (4, 2, (5,)), (26, 6, (0, 3, 30))]


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,lost", FUZZ)
def test_fuzz_against_the_oracle(cuda, swec, tmp_path, k, m, lost):
    """Random damage of 1-3 present shards per column, up to and past the radius, at file and device level."""
    ec = swec.erasure_coding
    torch = cuda
    length = 6_000 + 7
    rng = np.random.default_rng(k * 1000 + m * 10 + len(lost))
    shards = random_set(k, m, length, int(rng.integers(1 << 30)))
    present = mask(k + m, lost)
    ids = [i for i in range(k + m) if present[i]]
    for col in np.sort(rng.choice(length, size=length // 3, replace=False)):
        damage(shards, [col], rng, rng.choice(ids, size=int(rng.integers(1, 4)), replace=False))
    enc = ec.Encoder(k, m, device=0)
    for radius in (0, 1, 2):
        want, wrep = checked_rebuild(shards, k, m, present, radius)
        base = str(tmp_path / ("f%d" % radius))
        write_set(base, shards, lost=lost)
        rep = ec.rebuild_ec_files_checked(base, ctx=ec.ECContext(k, m), radius=radius)
        assert rep == {"rebuilt": list(lost), **wrep}, radius
        for i in lost:
            assert (np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) == want[i]).all(), (radius, i)
        for shift in (0, 3):
            bufs = [torch.zeros(length + 16, dtype=torch.uint8, device="cuda") for _ in range(k + m)]
            for i, b in enumerate(bufs):
                if present[i]:
                    b[shift:shift + length] = torch.from_numpy(shards[i]).cuda()
            got = enc.reconstruct_checked_device([b.data_ptr() + shift for b in bufs], present, length, radius=radius)
            assert got == {key: v for key, v in wrep.items() if key != "ok"}, (radius, shift)
            for i in range(k + m):
                back = bufs[i][shift:shift + length].cpu().numpy()
                assert (back == (want[i] if i in lost else shards[i])).all(), (radius, shift, i)
                assert (bufs[i][:shift] == 0).all() and (bufs[i][shift + length:] == 0).all(), (radius, shift, i)


@pytest.mark.gpu
def test_full_size_shards_in_hbm(cuda, swec):
    """13 x 3 GiB present shards plus one lost, in HBM, damaged in three present shards, checked by digest."""
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

    def digest(s):
        d = C.c_uint64(0)
        swec._native.check(L.swec_digest_device(0, s.data_ptr(), n, C.byref(d), None))
        return d.value

    want0 = digest(shards[0])
    ptrs = [s.data_ptr() for s in shards]
    present = [0] + [1] * 13
    run = 1_500_000_000
    shards[3][run:run + (1 << 20)] ^= 0x11          # 1 MiB run in an information shard
    shards[9][n - 1] ^= 0x80                        # the last byte of another
    shards[12][2 * GIB] ^= 0xFF                     # a check shard
    torch.cuda.synchronize()
    damaged = [digest(s) for s in shards[1:]]
    shards[0].zero_()
    rep = enc.reconstruct_checked_device(ptrs, present, n)
    assert rep["damaged_columns"] == (1 << 20) + 2 and rep["uncorrectable_columns"] == 0
    assert rep["shards"] == {3: (1 << 20, run, run + (1 << 20) - 1), 9: (1, n - 1, n - 1), 12: (1, 2 * GIB, 2 * GIB)}
    assert digest(shards[0]) == want0
    assert [digest(s) for s in shards[1:]] == damaged         # present shards are only read
    shards[0].zero_()
    enc.reconstruct_device(ptrs, present, n)
    enc.synchronize()
    assert digest(shards[0]) != want0                         # plain rebuild copies the damage
    del shards
    torch.cuda.empty_cache()
