"""Repair through the mounted volume: swec_ec_volume_repair_needle_damage (Python EcVolume.repair_needle_damage).

Expected values come from the calls it joins and from the existing oracles, never from the call itself:
- the composition: locate_needle_damage on the handle, then swec_repair_ec_damage by path, then scrub_needles over the
  repaired copy, on a second copy of the same damaged set; shard files, report, ranges, needles, unowned and findings
  must agree;
- test_needle_damage.handle_expected (damage_oracle.decode_columns through LocateData) for the report and the needles;
- the original .dat image for the bytes the reads return after the call;
- a miscorrection built from a weight-5 codeword of the code (oracle.rs_numpy), and checked with the oracle decoder.

cpu: argument rules and their order, each failing before any device work; the file checks; a handle opened with
device < 0; nothing opened for writing on any of those failures.
"""
from __future__ import annotations

import ctypes as C
import os
import re
import shutil
import stat
import sys
import tempfile
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import damage_oracle as do  # noqa: E402
import needle_oracle as no  # noqa: E402
import test_file_pipeline_exhaustive as tfe  # noqa: E402
import test_needle_damage as tnd  # noqa: E402

from oracle import rs_numpy as rn  # noqa: E402

GIB, MIB = tnd.GIB, tnd.MIB
CHECK_KEYS = ("status", "range_index", "data_size", "crc_got", "crc_want", "legacy_crc")
NEEDLE_OK, NEEDLE_BAD_CRC = 0, 3


# ---------------------------------------------------------------------------------------------- CPU


def raw_repair(swec, vol, radius=1, report=True, ranges_cap=0, needles_cap=0, needles=True, checks=True, unowned=True,
               handle=True):
    from seaweedfs_b200._native import DamageRange, DamageReport, NeedleCheck, NeedleDamage
    L = swec.lib()
    rep, n, nn, ok = DamageReport(), C.c_int(0), C.c_int(0), C.c_int(0)
    arr = (NeedleDamage * max(1, needles_cap))() if needles else None
    chk = (NeedleCheck * max(1, needles_cap))() if checks else None
    rng = (DamageRange * max(1, ranges_cap))()
    un = (C.c_uint64 * 2)() if unowned else None
    rc = L.swec_ec_volume_repair_needle_damage(vol._h if handle else None, radius, C.byref(rep) if report else None, rng,
                                               ranges_cap, C.byref(n), arr, chk, needles_cap, C.byref(nn), un, C.byref(ok))
    return rc, nn.value, ok.value, (arr, chk)


def shard_state(base, total=14):
    paths = [base + ".ec%02d" % i for i in range(total)]
    return {p: (open(p, "rb").read(), os.stat(p).st_mtime_ns) for p in paths if os.path.exists(p)}


def test_argument_rules_and_their_order(swec, tmp_path):
    """The rules of swec_ec_volume_locate_needle_damage in its order, the checks rule among the needle rules, then a
    handle without a device: nothing runs on a device and no shard file changes."""
    ec = swec.erasure_coding
    base = tnd.cpu_volume(tmp_path)
    before = shard_state(base)
    vol = ec.EcVolume(base, device=-1)
    L = swec.lib()

    def last():
        return L.swec_last_error()

    assert raw_repair(swec, vol, needles_cap=-1)[0] == -1
    assert raw_repair(swec, vol, needles_cap=3, needles=False)[0] == -1 and b"needles" in last()
    assert raw_repair(swec, vol, unowned=False)[0] == -1 and b"unowned" in last()
    # the new rule: checks NULL only with needles_cap 0, after the rules it joins and before every later rule
    assert raw_repair(swec, vol, needles_cap=3, checks=False)[0] == -1 and b"checks" in last()
    assert raw_repair(swec, vol, needles_cap=3, checks=False, unowned=False)[0] == -1 and b"unowned" in last()
    assert raw_repair(swec, vol, needles_cap=3, checks=False, handle=False)[0] == -1 and b"checks" in last()
    assert raw_repair(swec, vol, needles_cap=3, checks=False, radius=7)[0] == -1 and b"checks" in last()
    assert raw_repair(swec, vol, handle=False)[0] == -1 and b"NULL" in last()
    assert raw_repair(swec, vol, radius=7, unowned=False)[0] == -1 and b"unowned" in last()
    assert raw_repair(swec, vol, radius=7)[0] == -1 and b"radius" in last()
    assert raw_repair(swec, vol, radius=3)[0] == -1 and b"radius" in last()
    assert raw_repair(swec, vol, report=False)[0] == -1
    assert raw_repair(swec, vol, ranges_cap=2)[0] == -7         # ranges given: every check passes
    assert raw_repair(swec, vol, needles_cap=0, checks=False)[0] == -7
    assert raw_repair(swec, vol, needles_cap=4)[0] == -7
    assert b"device < 0" in last()
    with pytest.raises(swec._native.SwecError) as e:
        vol.repair_needle_damage()
    assert e.value.status == -7
    vol.close()
    assert shard_state(base) == before


def test_radius_against_the_parity_count(swec, tmp_path):
    """RS(6,3) takes radius 1 and refuses radius 2 (2t <= m), like the locate call on the same handle."""
    ec = swec.erasure_coding
    base = tnd.cpu_volume(tmp_path, k=6, m=3)
    import json
    vif = json.load(open(base + ".vif"))
    assert vif["ecShardConfig"] == {"dataShards": 6, "parityShards": 3}
    vol = ec.EcVolume(base, device=-1)
    assert raw_repair(swec, vol, radius=2)[0] == -1 and b"radius" in swec.lib().swec_last_error()
    assert tnd.raw_handle_call(swec, vol, radius=2) == -1
    assert raw_repair(swec, vol, radius=1)[0] == -7
    vol.close()


def test_file_checks_before_the_device(swec, tmp_path):
    """A shard that is not local, then unequal lengths, each before the device check, with nothing opened for
    writing: the files keep their bytes and mtimes."""
    ec = swec.erasure_coding
    base = tnd.cpu_volume(tmp_path)
    os.rename(base + ".ec12", base + ".ec12.away")
    vol = ec.EcVolume(base, device=-1)
    with pytest.raises(swec._native.SwecError) as e:
        vol.repair_needle_damage()
    assert e.value.status == -2 and ".ec12" in str(e.value)
    vol.close()
    os.rename(base + ".ec12.away", base + ".ec12")
    with open(base + ".ec03", "r+b") as f:
        f.truncate(os.path.getsize(base + ".ec03") - 1)
    before = shard_state(base)
    vol = ec.EcVolume(base, device=-1)
    with pytest.raises(swec._native.SwecError) as e:
        vol.repair_needle_damage()
    assert e.value.status == -6
    # both rules come before the device: the same order as the locate call on the same handle
    assert tnd.raw_handle_call(swec, vol) == -6
    vol.close()
    assert shard_state(base) == before


# ---------------------------------------------------------------------------------------------- GPU helpers


def clone(base, where):
    """A copy of the volume's shard, index and .vif files under `where`; returns its base."""
    os.makedirs(where, exist_ok=True)
    d, name = os.path.split(base)
    for f in os.listdir(d):
        if f.startswith(name + ".") and not f.endswith((".dat", ".idx")):
            shutil.copy2(os.path.join(d, f), os.path.join(where, f))
    return os.path.join(where, name)


def data_range(rec):
    """.dat offsets of the Data bytes of a record written by needle_oracle.write_record (no optional fields)."""
    _, off, size = rec
    return off + 20, off + 20 + max(0, size - 5)


def in_data(owners, live, d):
    """The index of the live record whose Data holds .dat offset d, or -1."""
    j = owners(d)
    if j < 0:
        return -1
    lo, hi = data_range(live[j])
    return j if lo <= d < hi else -1


def data_column(walk, live, shards, start=1000):
    """A column x >= start whose byte in each data shard of `shards` lies in the Data of a distinct live record;
    returns (x, [record index per shard])."""
    owners = tnd.Owners(live)
    for x in range(start, start + 200_000, 97):
        js = [in_data(owners, live, walk(s, x)) for s in shards]
        if all(j >= 0 for j in js) and len(set(js)) == len(js):
            return x, js
    raise AssertionError("no column with Data in every shard")


def miscorrecting_errors(k, m, flipped, blamed):
    """Error values at the shards `flipped` (3 of them) such that radius-2 decoding blames the 2 shards `blamed`
    instead: the restriction of the codeword supported on flipped + blamed, which the code's distance 5 makes unique
    up to a scalar.  Returns {shard: value}, checked against the oracle decoder."""
    support = sorted(flipped + blamed)
    gen = rn.build_matrix(k, k + m)
    data = [s for s in support if s < k]
    zero = [r for r in range(k, k + m) if r not in support]
    assert len(zero) == len(data) - 1
    # data values at `data` (the first fixed to 1) that make every parity row outside the support zero
    a = np.array([[gen[r][s] for s in data[1:]] for r in zero], dtype=np.uint8)
    b = np.array([[gen[r][data[0]]] for r in zero], dtype=np.uint8)
    rest = rn.mat_mul(rn.mat_inv(a), b)[:, 0]
    vec = np.zeros(k, dtype=np.uint8)
    vec[data[0]] = 1
    for s, v in zip(data[1:], rest):
        vec[s] = v
    word = rn.encode(k, m, [np.array([v], dtype=np.uint8) for v in vec])
    full = [int(v) for v in vec] + [int(p[0]) for p in word]
    assert [s for s in range(k + m) if full[s]] == support
    errors = {s: full[s] for s in flipped}
    col = [np.zeros(1, dtype=np.uint8) for _ in range(k + m)]
    for s, v in errors.items():
        col[s][0] = v
    _, x, y, _, _, _ = do.decode_columns(col, k, m, 2)
    assert sorted([int(x[0]), int(y[0])]) == sorted(blamed)
    return errors


def flip_at(base, shard, x, value):
    tnd.flip_file(base + ".ec%02d" % shard, x, value)


def findings(errors):
    """{needle id: text} of scrub_needles' needle findings."""
    out = {}
    for e in errors:
        mm = re.match(r"needle (\d+) on volume \d+: (.*)", e)
        if mm:
            out[int(mm[1])] = mm[2]
    return out


def strip_checks(needles):
    return [{key: v for key, v in r.items() if key not in CHECK_KEYS} for r in needles]


def new_volume(swec, tmp_path, name, k=10, m=4, seed=30):
    tmp_path.mkdir(parents=True, exist_ok=True)
    base, dat, live = tnd.generated_volume(swec, tmp_path, name, k=k, m=m, seed=seed)
    return base, dat, live, tnd.Striping(k, len(dat), GIB, MIB)


# ---------------------------------------------------------------------------------------------- GPU


SHAPES = [(10, 4, 1), (10, 4, 2), (6, 3, 1), (20, 12, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,radius", SHAPES)
def test_same_as_the_composition(cuda, swec, tmp_path, k, m, radius):
    """Two copies of one damaged set: the new call on one, and on the other locate_needle_damage, repair_ec_damage by
    path and scrub_needles.  Same shard files, report, ranges, needles, unowned and findings; the report and needles
    are also the oracle's."""
    ec = swec.erasure_coding
    base, dat, live, walk = new_volume(swec, tmp_path / "a", "1", k, m, seed=31 + k + radius)
    rng = np.random.default_rng(k * 10 + radius)
    for r in rng.choice(len(live), 12, replace=False):          # one shard in a column, inside Data
        lo, hi = data_range(live[int(r)])
        if hi > lo:
            i, x = walk.shard_pos(int(rng.integers(lo, hi)))
            flip_at(base, i, x, int(rng.integers(1, 256)))
    for start in (5000, 60_000):                                  # two data shards in a column
        x, _ = data_column(walk, live, [0, 1], start)
        flip_at(base, 0, x, 0x21)
        flip_at(base, 1, x, 0x12)
    flip_at(base, k + 1, 777, 0x08)                               # parity alone
    silent = set()
    if radius == 2:                                               # three shards: a miscorrection
        x, _ = data_column(walk, live, [1, 2], 90_000)
        for s, v in miscorrecting_errors(k, m, [0, 3, k], [1, 2]).items():
            flip_at(base, s, x, v)
        # the byte of data shard 0 stays wrong and is not blamed: no call names its needle
        a = tnd.Owners(live)(walk(0, x))
        silent = {live[a][0]} if a >= 0 else set()
    other = clone(base, str(tmp_path / "b"))
    vol = ec.EcVolume(base)
    shard_dat_size = vol.info()["shard_dat_size"]
    want = tnd.handle_expected(base, k, m, radius, live, shard_dat_size)
    res = vol.repair_needle_damage(radius=radius)
    tnd.handle_compare(res, want, live, k=k)
    vol.close()

    vb = ec.EcVolume(other)
    loc = vb.locate_needle_damage(radius=radius)
    rep = ec.repair_ec_damage(other, radius=radius)
    _, _, errors = vb.scrub_needles(3)
    vb.close()
    for i in range(k + m):
        assert open(base + ".ec%02d" % i, "rb").read() == open(other + ".ec%02d" % i, "rb").read(), i
    assert {key: v for key, v in res.items() if key not in ("ok", "needles")} == \
        {key: v for key, v in loc.items() if key not in ("ok", "needles")}
    assert strip_checks(res["needles"]) == loc["needles"]
    assert {key: v for key, v in rep.items() if key != "ok"} == {key: v for key, v in loc.items() if key in rep and key != "ok"}
    assert res["uncorrectable_columns"] > 0 or radius == 2

    found = findings(errors)
    named = {r["needle_id"]: r for r in res["needles"]}
    assert res["n_needles"] == len(named)
    assert {n for n, r in named.items() if r["status"] != NEEDLE_OK} == set(found) & set(named)
    assert set(found) - set(named) <= silent
    for nid, r in named.items():
        if r["status"] == NEEDLE_BAD_CRC:
            mm = re.search(r"got ([0-9a-f]{8}), want ([0-9a-f]{8})", found[nid])
            assert (r["crc_got"], r["crc_want"]) == (int(mm[1], 16), int(mm[2], 16))
        elif r["status"] == NEEDLE_OK:
            lo = r["offset"]
            assert r["data_size"] == int.from_bytes(dat[lo + 16:lo + 20].tobytes(), "big")
    assert res["ok"] == (rep["ok"] and not set(found) & set(named))
    if radius == 1:
        assert not res["ok"]


@pytest.mark.gpu
def test_one_wrong_shard_per_column(cuda, swec, tmp_path):
    """Every named needle re-checks ok, ok = 1, a second call finds nothing, and the reads return the records of the
    original .dat."""
    ec = swec.erasure_coding
    base, dat, live, walk = new_volume(swec, tmp_path, "2")
    rng = np.random.default_rng(2)
    picked = [live[int(r)] for r in rng.choice(len(live), 20, replace=False)]
    for rec in picked:
        lo, hi = data_range(rec)
        i, x = walk.shard_pos(rec[1] + 4 if hi <= lo else int(rng.integers(lo, hi)))
        flip_at(base, i, x, int(rng.integers(1, 256)))
    vol = ec.EcVolume(base)
    res = vol.repair_needle_damage()
    assert res["ok"] and res["uncorrectable_columns"] == 0
    assert {r["needle_id"] for r in res["needles"]} == {r[0] for r in picked}
    assert all(r["status"] == NEEDLE_OK and r["damaged_bytes"] >= 1 for r in res["needles"])
    again = vol.repair_needle_damage()
    assert again["ok"] and again["damaged_columns"] == 0 and again["n_needles"] == 0 and again["needles"] == []
    for got, rec in zip(vol.read_needles([r[0] for r in picked]), picked):
        n = no.actual_size(rec[2], 3)
        assert got["status"] == "SWEC_OK" and bytes(got["bytes"][:n]) == dat[rec[1]:rec[1] + n].tobytes()
    vol.close()


@pytest.mark.gpu
def test_two_wrong_data_shards_at_radius_1(cuda, swec, tmp_path):
    """The column is uncorrectable and keeps its bytes; its needles have uncorrectable bytes, the damaged ones re-check
    as a bad CRC, and ok = 0."""
    ec = swec.erasure_coding
    base, dat, live, walk = new_volume(swec, tmp_path, "3")
    x, js = data_column(walk, live, [0, 1], 20_000)
    flip_at(base, 0, x, 0x5A)
    flip_at(base, 1, x, 0xA5)
    column = [open(base + ".ec%02d" % i, "rb").read()[x] for i in range(14)]
    vol = ec.EcVolume(base)
    res = vol.repair_needle_damage(radius=1)
    assert not res["ok"] and res["uncorrectable_columns"] == 1 and res["damaged_columns"] == 1
    assert [open(base + ".ec%02d" % i, "rb").read()[x] for i in range(14)] == column
    by_id = {r["needle_id"]: r for r in res["needles"]}
    for j in js:
        r = by_id[live[j][0]]
        assert r["uncorrectable_bytes"] > 0 and r["damaged_bytes"] == 0 and r["status"] == NEEDLE_BAD_CRC
    assert all(r["uncorrectable_bytes"] > 0 for r in res["needles"])
    # nothing changed, so the call again, through the C ABI: checks[i] names needles[i]
    rc, n_needles, ok, (arr, chk) = raw_repair(swec, vol, needles_cap=64)
    assert (rc, n_needles, ok) == (0, res["n_needles"], 0)
    assert [(c.needle_id, c.offset, c.size, c.status) for c in chk[:n_needles]] == \
        [(r["needle_id"], r["offset"], r["size"], r["status"]) for r in res["needles"]]
    assert [(a.needle_id, a.uncorrectable_bytes) for a in arr[:n_needles]] == \
        [(r["needle_id"], r["uncorrectable_bytes"]) for r in res["needles"]]
    vol.close()


@pytest.mark.gpu
def test_three_wrong_shards_at_radius_2_miscorrected(cuda, swec, tmp_path):
    """Three wrong shards in one column of RS(10,4): radius 2 rewrites it into another codeword, and the report calls it
    corrected.  The needles whose bytes the miscorrection rewrote re-check as a bad CRC, and ok = 0."""
    ec = swec.erasure_coding
    base, dat, live, walk = new_volume(swec, tmp_path, "4")
    x, js = data_column(walk, live, [1, 2], 40_000)
    for s, v in miscorrecting_errors(10, 4, [0, 3, 10], [1, 2]).items():
        flip_at(base, s, x, v)
    vol = ec.EcVolume(base)
    res = vol.repair_needle_damage(radius=2)
    assert res["uncorrectable_columns"] == 0 and res["damaged_columns"] == 1
    assert set(res["shards"]) == {1, 2}
    assert not res["ok"]
    named = {r["needle_id"]: r for r in res["needles"]}
    assert set(named) == {live[j][0] for j in js}
    assert all(r["status"] == NEEDLE_BAD_CRC and r["damaged_bytes"] == 1 for r in named.values())
    # the same call again finds a codeword in that column: the damage is now silent to the code
    again = vol.repair_needle_damage(radius=2)
    assert again["damaged_columns"] == 0 and again["ok"]
    vol.close()


@pytest.mark.gpu
def test_parity_only_damage(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    base, _, _, _ = new_volume(swec, tmp_path, "5")
    clean = {i: open(base + ".ec%02d" % i, "rb").read() for i in (11, 13)}
    flip_at(base, 11, 4321, 0x10)
    flip_at(base, 13, 100_000, 0x01)
    vol = ec.EcVolume(base)
    res = vol.repair_needle_damage()
    assert res["ok"] and res["n_needles"] == 0 and res["needles"] == [] and res["unowned"] == [0, 0]
    assert res["damaged_columns"] == 2 and set(res["shards"]) == {11, 13}
    assert {i: open(base + ".ec%02d" % i, "rb").read() for i in (11, 13)} == clean
    vol.close()


@pytest.mark.gpu
def test_clean_set_opens_nothing_for_writing(cuda, swec, tmp_path):
    ec = swec.erasure_coding
    base, _, _, _ = new_volume(swec, tmp_path, "6")
    for i in range(14):
        os.utime(base + ".ec%02d" % i, ns=(10**18, 10**18))
    before = shard_state(base)
    plain = ec.locate_ec_damage(base)
    vol = ec.EcVolume(base)
    with tfe.DirectWatch(str(tmp_path)) as w:
        res = vol.repair_needle_damage()
    assert res["ok"] and res["n_needles"] == 0 and res["needles"] == [] and res["unowned"] == [0, 0]
    assert {key: res[key] for key in plain} == plain
    assert all(mode == os.O_RDONLY for mode, _ in w.seen)
    assert shard_state(base) == before
    vol.close()


@pytest.mark.gpu
def test_needles_cap(cuda, swec, tmp_path):
    """A cap below the number of named needles, and 0 with checks NULL: n_needles counts them all, and ok still covers
    the needles past the cap (here the two a radius-2 miscorrection rewrites, which have the largest ids)."""
    ec = swec.erasure_coding
    base, dat, live, walk = new_volume(swec, tmp_path, "7")
    x, js = data_column(walk, live, [1, 2], 40_000)
    for s, v in miscorrecting_errors(10, 4, [0, 3, 10], [1, 2]).items():
        flip_at(base, s, x, v)
    first = min(live[j][0] for j in js)
    early = [r for r in live if r[0] < first and data_range(r)[1] > data_range(r)[0]][:6]
    assert len(early) == 6
    for rec in early:
        i, xx = walk.shard_pos(data_range(rec)[0])
        flip_at(base, i, xx, 0x77)
    copy = clone(base, str(tmp_path / "copy"))
    vol = ec.EcVolume(base)
    res = vol.repair_needle_damage(radius=2, max_needles=len(early))
    assert res["n_needles"] == len(early) + 2 and [r["needle_id"] for r in res["needles"]] == [r[0] for r in early]
    assert all(r["status"] == NEEDLE_OK for r in res["needles"]) and not res["ok"]
    vol.close()
    vc = ec.EcVolume(copy)
    rc, n_needles, ok, _ = raw_repair(swec, vc, radius=2, needles_cap=0, needles=False, checks=False)
    assert (rc, n_needles, ok) == (0, len(early) + 2, 0)
    vc.close()
    for i in range(14):
        assert open(base + ".ec%02d" % i, "rb").read() == open(copy + ".ec%02d" % i, "rb").read(), i


@pytest.mark.gpu
def test_reads_on_the_same_handle(cuda, swec, tmp_path):
    """Reads issued from another thread while the call runs return each needle as it was before the call or as
    corrected, never a mix; after the call the reads return the original records."""
    ec = swec.erasure_coding
    base, dat, live, walk = new_volume(swec, tmp_path, "8")
    rng = np.random.default_rng(8)
    picked = [live[int(r)] for r in rng.choice(len(live), 30, replace=False) if data_range(live[int(r)])[1] > data_range(live[int(r)])[0]]
    for rec in picked:                                   # two bytes per needle, in two shards where it spans them
        lo, hi = data_range(rec)
        for d in (lo, hi - 1):
            i, x = walk.shard_pos(d)
            flip_at(base, i, x, 0x3C)
    ids = [r[0] for r in picked]
    vol = ec.EcVolume(base)
    pre = {r["id"]: bytes(r["bytes"]) for r in vol.read_needles(ids)}
    seen, stop = [], threading.Event()

    def reader():
        while not stop.is_set():
            seen.append({r["id"]: bytes(r["bytes"]) for r in vol.read_needles(ids)})

    t = threading.Thread(target=reader)
    t.start()
    try:
        res = vol.repair_needle_damage()
    finally:
        stop.set()
        t.join()
    assert res["ok"] and {r["needle_id"] for r in res["needles"]} == set(ids)
    post = {r["id"]: bytes(r["bytes"]) for r in vol.read_needles(ids)}
    for rec in picked:
        n = no.actual_size(rec[2], 3)
        assert post[rec[0]][:n] == dat[rec[1]:rec[1] + n].tobytes() and pre[rec[0]] != post[rec[0]]
    assert seen
    for snap in seen:
        for nid, b in snap.items():
            assert b in (pre[nid], post[nid]), nid
    vol.close()


@pytest.mark.gpu
def test_refused_write_fails_before_anything_is_written(cuda, swec, tmp_path):
    """A blamed shard that cannot be opened for writing fails the call with SWEC_ERR_IO, and no shard is written."""
    if os.geteuid() == 0:
        pytest.skip("root opens a read-only file for writing")
    ec = swec.erasure_coding
    base, dat, live, walk = new_volume(swec, tmp_path, "9")
    for rec in live[10:40:5]:
        lo, hi = data_range(rec)
        if hi > lo:
            i, x = walk.shard_pos(lo)
            flip_at(base, i, x, 0x01)
    flip_at(base, 12, 999, 0x02)
    os.chmod(base + ".ec12", stat.S_IRUSR)
    before = shard_state(base)
    vol = ec.EcVolume(base)
    try:
        with pytest.raises(swec._native.SwecError) as e:
            vol.repair_needle_damage()
        assert e.value.status == -4 and ".ec12" in str(e.value)
        assert shard_state(base) == before
    finally:
        os.chmod(base + ".ec12", stat.S_IRUSR | stat.S_IWUSR)
        vol.close()


@pytest.fixture(scope="module")
def odirect(tmp_path_factory):
    d, tried, strict = tfe.direct_dir(tmp_path_factory.mktemp("odirect"))
    yield d, tried
    if d and d.startswith(os.path.join(tfe.ROOT, ".pytest_cache")):
        shutil.rmtree(d, ignore_errors=True)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_file_direct_io(cuda, swec, odirect, mode):
    """file_direct_io 0-3: the repaired files equal the original shards, and the write side uses an O_DIRECT descriptor
    exactly when bit 1 is set."""
    where, tried = odirect
    if where is None:
        pytest.skip("no filesystem here accepts O_DIRECT: " + ", ".join(tried))
    ec = swec.erasure_coding
    root = tempfile.mkdtemp(prefix="repair-mode%d-" % mode, dir=where)
    tfe.set_option(swec, b"file_direct_io", mode)
    try:
        from pathlib import Path
        base, dat, live, walk = new_volume(swec, Path(root), "10", seed=40 + mode)
        clean = {i: open(base + ".ec%02d" % i, "rb").read() for i in range(14)}
        rng = np.random.default_rng(mode)
        vol = ec.EcVolume(base)
        seen = set()
        # a repair of a small set holds its write descriptors for milliseconds: damage and repair again until the
        # watch has seen them
        for _ in range(8):
            for r in rng.choice(len(live), 10, replace=False):
                lo, hi = data_range(live[int(r)])
                if hi > lo:
                    i, x = walk.shard_pos(int(rng.integers(lo, hi)))
                    flip_at(base, i, x, 0x44)
            flip_at(base, 10, int(rng.integers(0, len(clean[10]))), 0x01)
            with tfe.DirectWatch(root) as w:
                res = vol.repair_needle_damage()
            seen |= w.seen
            assert res["ok"] and res["damaged_columns"] >= 2
            assert {i: open(base + ".ec%02d" % i, "rb").read() for i in range(14)} == clean
            if any(m != os.O_RDONLY and dd == bool(mode & 2) for m, dd in seen):
                break
        vol.close()
        writes = {dd for m, dd in seen if m != os.O_RDONLY}
        assert writes, (mode, sorted(seen))
        assert (True in writes) == bool(mode & 2), (mode, sorted(seen), tfe.fs_type(where))
    finally:
        tfe.set_option(swec, b"file_direct_io", tfe.default_direct())
        shutil.rmtree(root, ignore_errors=True)
