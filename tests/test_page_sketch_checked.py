"""Damage located from the sketches of a set with lost shards, and the sketches its rebuild must produce
(include/swec.h, swec_locate_sketch_damage_checked).

CPU: a checked page oracle (damage_oracle's errors-and-erasures column decode of the sketch bytes, merged per page) that
meets the per-page guarantee, with m replaced by c, for every loss pattern and damaged set of RS(3,2) and RS(6,3), and
whose rebuilt sketches are those of the true lost shard on clean and blamed pages and of the plain rebuild on
uncorrectable ones; the argument rules on a device-less encoder.
GPU: the call against the oracle on a damage corpus times loss patterns, against swec_locate_sketch_damage with nothing
lost, on clean sets, on 786,432-page sketch arrays, and end to end on shard files that each sit in a directory of
their own: repair the blamed pages at their holders, rebuild, and check the rebuilt shard against the prediction.
"""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

import damage_oracle as do
from oracle import rs_numpy as rn
from test_page_sketch import (PAGE, _corpus, _damage, _device_sketches, _generate, _read_page, _write_page, clean_set,
                              mask_of, sketch)


def _set(L, **opts):
    for name, value in opts.items():
        assert L.swec_set_option(name.encode(), int(value)) == 0, (name, value)


@pytest.fixture(scope="module", autouse=True)
def inline_compiles(swec):
    """The sketch arrays here are short, so the applies of the loss patterns' matrices would queue their run-time
    kernels for the background compiler, which would still be compiling them while later modules count compiles.
    jit_min_bytes 0 compiles them inline, within this module; the documented defaults come back afterwards."""
    L = swec.lib()
    _set(L, jit_min_bytes=0)
    try:
        yield L
    finally:
        _set(L, jit=1, jit_min_bytes=64 << 20)


# ---------------------------------------------------------------------------------------------------------- oracle

def _bytes(s):
    return np.ascontiguousarray(s, dtype="<u8").view(np.uint8)


def checked_oracle(sketches, k: int, m: int, radius: int):
    """(flagged pages [(page, blamed mask, uncorrectable)], {lost id: rebuilt sketch words}) of a set whose lost shards
    have sketch None, at radius t = min(radius, c // 2).  Column (g, l) of the sketches is byte 8g+l."""
    present = tuple(s is not None for s in sketches)
    info, checks, lost, _, r = do.punctured_rows(k, m, present)
    t = min(radius, len(checks) // 2)
    b = [None if s is None else _bytes(s) for s in sketches]
    plain = rn.apply_rows(r, [b[i] for i in info]) if lost else []
    if not checks:
        return [], {i: p.view("<u8").copy() for i, p in zip(lost, plain)}
    cols, a, bb, va, vb, ids = do.decode_columns(b, k, m, t, present)
    pages = {}
    for col, x, y, ex, ey in zip(cols.tolist(), a.tolist(), bb.tolist(), va.tolist(), vb.tolist()):
        mask, bad, errs = pages.get(col // 8, (0, False, []))
        if x < 0:
            bad = True
        else:
            mask |= 1 << int(ids[x])
            errs.append((col, x, ex))
            if y >= 0:
                mask |= 1 << int(ids[y])
                errs.append((col, y, ey))
        pages[col // 8] = (mask, bad, errs)
    out = []
    fixed = [p.copy() for p in plain]
    for g in sorted(pages):
        mask, bad, errs = pages[g]
        bad = bad or bin(mask).count("1") > t
        out.append((g, 0 if bad else mask, bad))
        if not bad:
            for col, pos, e in errs:
                if pos < k:           # an information error reached every rebuilt byte of its column
                    for x in range(len(lost)):
                        fixed[x][col] ^= rn.MUL[r[x][pos], e]
    return out, {i: f.view("<u8").copy() for i, f in zip(lost, fixed)}


def _per_shard(pages, n):
    per = {}
    for _, mask, _ in pages:
        for i in range(n):
            if mask >> i & 1:
                per[i] = per.get(i, 0) + 1
    return per


# ---------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("k,m", [(3, 2), (6, 3)])
def test_oracle_meets_the_guarantee_for_every_loss_and_damage(oracle, k, m):
    """Every loss pattern with c >= 1, every damaged set D of present shards with |D| <= c, every t <= c // 2: D exactly,
    uncorrectable, or flagged; and the rebuilt sketches are the true lost shard's on clean and blamed pages and the
    plain rebuild's on uncorrectable ones.  Page 0 of 2 is clean, page 1 damaged."""
    n = PAGE + 700
    shards = clean_set(k, m, n, 7 * k + m)
    rng = np.random.default_rng(k * 13 + m)
    for f in range(m):
        for lost in itertools.combinations(range(k + m), f):
            seed = int(rng.integers(0, 1 << 63))
            clean = [sketch(oracle, s, seed) for s in shards]
            pres = [i for i in range(k + m) if i not in lost]
            c = len(pres) - k
            for size in range(1, c + 1):
                for dset in itertools.combinations(pres, size):
                    bad = [s.copy() for s in shards]
                    for i in dset:
                        at = rng.choice(np.arange(PAGE, n), size=int(rng.integers(1, 30)), replace=False)
                        bad[i][at] ^= rng.integers(1, 256, len(at), dtype=np.uint8)
                    sk = [None if i in lost else (sketch(oracle, bad[i], seed) if i in dset else clean[i])
                          for i in range(k + m)]
                    # what the plain rebuild writes: the lost shards from the first k present shards as found
                    plain = rn.reconstruct(k, m, [None if i in lost else bad[i] for i in range(k + m)])
                    plain_sk = {i: sketch(oracle, plain[i], seed) for i in lost}
                    for t in range(0, c // 2 + 1):
                        got, rebuilt = checked_oracle(sk, k, m, t)
                        assert [p for p, _, _ in got] == [1], (lost, dset, t)
                        if size <= t:
                            assert got == [(1, mask_of(dset), False)], (lost, dset, t)
                        elif size <= c - t:
                            assert got == [(1, 0, True)], (lost, dset, t)
                        for i in lost:
                            assert rebuilt[i][0] == clean[i][0], (lost, dset, t, i)
                            want = plain_sk[i][1] if got[0][2] else clean[i][1]
                            if size <= c - t:   # beyond that the blame, and so the correction, can be wrong
                                assert rebuilt[i][1] == want, (lost, dset, t, i)


def test_oracle_with_nothing_checkable_is_the_plain_rebuild(oracle):
    k, m = 3, 2
    shards = clean_set(k, m, 2 * PAGE, 1)
    sk = [sketch(oracle, s, 5) for s in shards]
    got, rebuilt = checked_oracle([sk[0], None, sk[2], None, sk[4]], k, m, 2)
    assert got == [] and sorted(rebuilt) == [1, 3]
    assert (rebuilt[1] == sk[1]).all() and (rebuilt[3] == sk[3]).all()


def _raw(L, enc_h, sketches, shard_len, radius, pages, cap, n, per, outs, ok):
    return L.swec_locate_sketch_damage_checked(enc_h, sketches, shard_len, radius, pages, cap, n, per, outs, ok)


def test_argument_rules_before_any_device_work(swec):
    from seaweedfs_b200._native import SketchPage
    ec = swec.erasure_coding
    L = swec.lib()
    enc = ec.Encoder(3, 2, device=-1)
    words = [np.zeros(2, dtype=np.uint64) for _ in range(5)]
    arr = (C.c_void_p * 5)(*[w.ctypes.data for w in words])
    outs = (C.c_void_p * 5)()
    pages, n, per, ok = (SketchPage * 4)(), C.c_int64(0), (C.c_uint64 * 32)(), C.c_int(0)
    args = dict(enc_h=enc._h, sketches=arr, shard_len=PAGE + 1, radius=1, pages=pages, cap=4, n=C.byref(n), per=per,
                outs=outs, ok=C.byref(ok))

    def call(**over):
        return _raw(L, **{**args, **over})
    assert call(enc_h=None) == -1
    assert call(sketches=None) == -1
    assert call(n=None) == -1 and call(ok=None) == -1
    assert call(shard_len=-1) == -1
    assert call(cap=-1) == -1 and call(pages=None) == -1
    assert call(radius=-1) == -1 and call(radius=3) == -1
    two_lost = (C.c_void_p * 5)(words[0].ctypes.data, None, words[2].ctypes.data, None, words[4].ctypes.data)
    three_lost = (C.c_void_p * 5)(words[0].ctypes.data, None, None, None, words[4].ctypes.data)
    assert call(sketches=three_lost) == -2                 # fewer than k sketches
    assert call(sketches=three_lost, radius=3) == -1       # argument errors first
    assert call(sketches=three_lost, cap=-1) == -1
    # then the device: radius 2 with m = 2 (c = 2) passes the argument check, as it is clamped to c // 2
    assert call(radius=2) == -7
    assert call(sketches=two_lost, radius=2) == -7
    assert call(pages=None, cap=0, per=None, outs=None) == -7
    assert call(shard_len=0) == -7
    assert call() == -7
    with pytest.raises(swec.SwecError) as e:
        enc.locate_sketch_damage_checked(words[:4] + [None], [PAGE + 1] * 3 + [PAGE + 2, None])
    assert e.value.name == "SWEC_ERR_SHARD_SIZE"
    with pytest.raises(swec.SwecError) as e:
        enc.locate_sketch_damage_checked([words[0], None, None, None, words[4]], PAGE + 1)
    assert e.value.name == "SWEC_ERR_TOO_FEW_SHARDS"
    with pytest.raises(swec.SwecError) as e:
        enc.locate_sketch_damage_checked(words[:4] + [None], PAGE + 1, radius=2)
    assert e.value.name == "SWEC_ERR_NO_DEVICE"


# ---------------------------------------------------------------------------------------------------------- GPU

def _losses(k, m):
    """name -> lost shard ids: none, one data, one parity, two mixed, and c = 0 (m lost, data and parity)."""
    return {"none": (), "one_data": (1,), "one_parity": (k,), "two_mixed": (2, k + 1),
            "c0": tuple([0] + list(range(k + 1, k + m)))}


def _check(res, want, rebuilt, k, m, what):
    assert res["pages"] == want, what
    assert res["n_flagged"] == len(want), what
    assert res["shard_pages"] == _per_shard(want, k + m), what
    assert sorted(res["rebuilt"]) == sorted(rebuilt), what
    for i, w in rebuilt.items():
        assert (res["rebuilt"][i] == w).all(), (what, i, np.flatnonzero(res["rebuilt"][i] != w)[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,radius", [(10, 4, 1), (10, 4, 2), (10, 4, 0), (6, 3, 1), (3, 2, 1), (20, 12, 1)])
def test_locate_equals_the_checked_oracle(swec, cuda, oracle, k, m, radius):
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    n = 6 * PAGE + 1234
    shards = clean_set(k, m, n, k + m + 1)
    rng = np.random.default_rng(radius * 37 + k)
    for lname, lost in _losses(k, m).items():
        c = m - len(lost)
        for name, spec in _corpus(k, m, n, rng).items():
            seed = int(rng.integers(0, 1 << 63))
            sk = _device_sketches(cuda, enc, _damage(shards, spec, rng), seed)
            sk = [None if i in lost else s for i, s in enumerate(sk)]
            want, rebuilt = checked_oracle(sk, k, m, radius)
            res = enc.locate_sketch_damage_checked(sk, n, radius=radius)
            _check(res, want, rebuilt, k, m, (lname, name))
            assert res["checks"] == c
            assert res["ok"] == (c >= 1 and not want), (lname, name)
            if c == 0:
                assert res["n_flagged"] == 0 and not res["ok"]
            if not lost and 2 * radius <= m:
                assert enc.locate_sketch_damage(sk, n, radius=radius) == \
                    {key: res[key] for key in ("ok", "n_flagged", "pages", "shard_pages")}, name


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", [(10, 4), (6, 3), (20, 12), (3, 2)])
def test_clean_sets_flag_nothing_and_predict_the_lost_shards(swec, cuda, k, m):
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    n = 5 * PAGE + 77
    true = _device_sketches(cuda, enc, clean_set(k, m, n, 3), 0xFEED)
    for lost in _losses(k, m).values():
        sk = [None if i in lost else s for i, s in enumerate(true)]
        for t in (0, 1, 2):
            res = enc.locate_sketch_damage_checked(sk, n, radius=t)
            assert res["n_flagged"] == 0 and res["pages"] == [] and res["shard_pages"] == {}
            assert res["ok"] == (len(lost) < m)
            assert sorted(res["rebuilt"]) == sorted(lost)
            for i in lost:
                assert (res["rebuilt"][i] == true[i]).all(), (lost, t, i)


@pytest.mark.gpu
def test_lost_sketches_not_asked_for_are_not_written(swec, cuda):
    from seaweedfs_b200._native import SketchPage
    k, m = 6, 3
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    n = 3 * PAGE
    true = _device_sketches(cuda, enc, clean_set(k, m, n, 9), 0xBEEF)
    present = [None if i in (1, 7) else s for i, s in enumerate(true)]
    arr = (C.c_void_p * (k + m))(*[None if s is None else s.ctypes.data for s in present])
    seven = np.full(3, 0x55, dtype=np.uint64)
    decoy = np.full(3, 0x66, dtype=np.uint64)
    outs = (C.c_void_p * (k + m))(*[seven.ctypes.data if i == 7 else decoy.ctypes.data if i == 0 else None
                                    for i in range(k + m)])
    pages, nf, ok = (SketchPage * 3)(), C.c_int64(-1), C.c_int(-1)
    assert swec.lib().swec_locate_sketch_damage_checked(enc._h, arr, n, 1, pages, 3, C.byref(nf), None, outs,
                                                        C.byref(ok)) == 0
    assert nf.value == 0 and ok.value == 1
    assert (seven == true[7]).all() and (decoy == 0x66).all()   # a present shard's entry is ignored
    assert swec.lib().swec_locate_sketch_damage_checked(enc._h, arr, n, 1, pages, 3, C.byref(nf), None, None,
                                                        C.byref(ok)) == 0
    assert swec.lib().swec_locate_sketch_damage_checked(enc._h, arr, 0, 1, None, 0, C.byref(nf), None, outs,
                                                        C.byref(ok)) == 0
    assert nf.value == 0 and ok.value == 1


@pytest.mark.gpu
def test_full_size_volume_with_two_lost_shards(swec, cuda):
    """786,432 pages per shard (a 30 GiB RS(10,4) volume): synthetic codeword sketch arrays with scattered errors on
    present shards, two shards lost, against the oracle."""
    k, m, pages = 10, 4, 786432
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    rng = np.random.default_rng(786432)
    data = [rng.integers(0, 256, 8 * pages, dtype=np.uint8) for _ in range(k)]
    words = [d.view("<u8") for d in data] + [p.view("<u8") for p in rn.encode(k, m, data)]
    lost = (4, 12)
    present = [i for i in range(k + m) if i not in lost]
    sk = [None if i in lost else words[i].copy() for i in range(k + m)]
    hit = {}   # page -> the present shards damaged there
    for g in rng.choice(pages, 300, replace=False):
        hit[int(g)] = [int(i) for i in rng.choice(present, int(rng.integers(1, 3)), replace=False)]
        for i in hit[int(g)]:
            b = sk[i][g:g + 1].view(np.uint8)
            b[int(rng.integers(0, 8))] ^= int(rng.integers(1, 256))
    want, rebuilt = checked_oracle(sk, k, m, 1)
    res = enc.locate_sketch_damage_checked(sk, pages * PAGE, radius=1)
    _check(res, want, rebuilt, k, m, "full")
    assert [g for g, _, _ in want] == sorted(hit)
    single = {g for g, ids in hit.items() if len(ids) == 1}
    assert single and len(single) < len(hit)
    # c = 2, t = 1: one damaged shard is blamed exactly, and the prediction is the true lost shard on every other page
    assert {(g, mask) for g, mask, bad in want if g in single} == {(g, 1 << hit[g][0]) for g in single}
    for i in lost:
        assert set(np.flatnonzero(res["rebuilt"][i] != words[i]).tolist()) <= set(hit) - single


def _shard_set(swec, root, k, m, seed):
    root.mkdir()
    return _generate(swec, root, k, m, seed)


def _rebuild_flow(swec, root, k, m, lost, damage, repair):
    """Lose `lost`, damage present files, sketch them, locate with the checked call, repair the blamed pages at their
    holders from k present shards outside the blame (when `repair`), then run the plain rebuild.  Returns (files,
    originals, result, rebuilt sketches of the lost files, base)."""
    ec = swec.erasure_coding
    base, dirs, files = _shard_set(swec, root, k, m, 100 + k)
    originals = [open(f, "rb").read() for f in files]
    n = len(originals[0])
    rng = np.random.default_rng(k + len(lost))
    for i in lost:
        os.unlink(files[i])
    for i, offs in damage.items():
        b = np.frombuffer(originals[i], dtype=np.uint8).copy()
        b[offs] ^= rng.integers(1, 256, len(offs), dtype=np.uint8)
        open(files[i], "wb").write(b.tobytes())
    seed = 0x5EED0000 + k
    sketches = [None if i in lost else ec.page_sketch_file(f, seed)[0] for i, f in enumerate(files)]
    lengths = [None if i in lost else os.path.getsize(f) for i, f in enumerate(files)]
    enc = ec.Encoder(k, m, device=0)
    res = enc.locate_sketch_damage_checked(sketches, lengths, radius=1)
    if repair:
        batch, targets = [], []
        for g, mask, bad in res["pages"]:
            assert not bad
            src = [i for i in range(k + m) if i not in lost and not mask >> i & 1][:k]
            assert len(src) == k
            item = [None] * (k + m)
            for i in src:
                item[i] = _read_page(files[i], g, n)
            batch.append(item)
            targets.append((g, mask))
        enc.reconstruct_batch(batch, data_only=False)
        for item, (g, mask) in zip(batch, targets):
            for i in range(k + m):
                if mask >> i & 1:
                    _write_page(files[i], g, item[i])
    # the file pipeline never waits for a compile: jit 0 keeps it from queueing one (see inline_compiles)
    _set(swec.lib(), jit=0)
    try:
        assert sorted(ec.rebuild_ec_files(base, dirs, ec.ECContext(k, m, device=0))) == sorted(lost)
    finally:
        _set(swec.lib(), jit=1)
    out = {i: ec.page_sketch_file(base + ec.ToExt(i), seed)[0] for i in lost}
    return files, originals, res, out, base


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,lost", [(10, 4, (3,)), (10, 4, (1, 12)), (6, 3, (0,))])
def test_check_repair_and_rebuild_a_balanced_set(swec, cuda, tmp_path, k, m, lost):
    """Locate from the present shards' sketches, repair the blamed pages where they lie, rebuild: every file is the
    original and the rebuilt shard has the predicted sketch.  Without the repair, the rebuilt shard's sketch differs
    from the prediction exactly on the pages blamed on an information shard."""
    ec = swec.erasure_coding
    pres = [i for i in range(k + m) if i not in lost]
    info, check = pres[0], pres[-1]   # an information shard and a check shard
    damage = {info: [5000, 5001], check: [3 * PAGE + 7], pres[1]: [8 * PAGE + 10]}
    files, originals, res, out, base = _rebuild_flow(swec, tmp_path / "a", k, m, lost, damage, repair=True)
    assert {g for g, _, _ in res["pages"]} == {1, 3, 8} and not res["ok"]
    assert res["pages"] == [(1, 1 << info, False), (3, 1 << check, False), (8, 1 << pres[1], False)]
    for i in range(k + m):
        path = base + ec.ToExt(i) if i in lost else files[i]
        assert open(path, "rb").read() == originals[i], i
    for i in lost:
        assert (out[i] == res["rebuilt"][i]).all(), i

    _, _, res2, out2, _ = _rebuild_flow(swec, tmp_path / "b", k, m, lost, damage, repair=False)
    assert res2["pages"] == res["pages"]
    on_info = {g for g, mask, _ in res2["pages"] if mask & ~(1 << check)}
    for i in lost:
        assert (res2["rebuilt"][i] == res["rebuilt"][i]).all()
        assert set(np.flatnonzero(out2[i] != res2["rebuilt"][i]).tolist()) == on_info, i
