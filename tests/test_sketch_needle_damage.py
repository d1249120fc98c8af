"""Which needles sketch-located EC damage hits, and the holder's sketch through the mounted volume:
swec_sketch_needle_damage, swec_ec_volume_sketch_needle_damage and swec_ec_volume_page_sketch.

Expected values share nothing with the method:
- attribution_oracle maps every byte of every attributed (page, data shard) to its .dat offset with a vectorised
  striping formula, and finds owners with numpy.searchsorted; on tiny geometries it is checked against a literal loop
  over the bytes with test_needle_damage's walk of encodeDatFile's blocks and its bisect owner;
- at full size the damaged bytes of a fully flagged data shard come from the closed form of how many bytes of [0, d)
  that shard holds;
- on a mounted volume, page-aligned damage makes the byte-level swec_ec_volume_locate_needle_damage the reference.

cpu: the oracle against the literal loop; every argument rule and the error order of the three calls, on device-less
handles.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

import needle_oracle as no
from oracle import rs_numpy as rn
from test_needle_damage import Owners, Striping, generated_volume, image
from test_page_sketch import PAGE, _device_sketches, _generate
from test_page_sketch_checked import inline_compiles  # noqa: F401  (autouse: the loss patterns compile inline)

MIB, GIB = 1 << 20, 1 << 30


# ---------------------------------------------------------------------------------------------- oracle side


def dat_offsets(k, i, x, large, small, large_rows, dat_end):
    """.dat offset of the shard offsets x of data shard i (-1: padding), for large_rows rows of large blocks."""
    x = np.asarray(x, dtype=np.int64)
    lb = large_rows * large
    y = x - lb
    d = np.where(x < lb, (x // large) * large * k + i * large + x % large,
                 lb * k + (y // small) * small * k + i * small + y % small)
    return np.where(d < dat_end, d, -1)


def encode_geometry(k, dat_size, large, small):
    return dict(large=large, small=small, large_rows=dat_size // (large * k), dat_end=dat_size)


def spans(records, version=3):
    """(offsets, ends, order): the records sorted by offset (a stable sort: the later entry last on a tie)."""
    order = sorted(range(len(records)), key=lambda j: records[j][1])
    offs = np.array([records[j][1] for j in order], dtype=np.int64)
    ends = np.array([records[j][1] + (no.actual_size(records[j][2], version) if records[j][2] >= 0 else 0)
                     for j in order], dtype=np.int64)
    return offs, ends, np.array(order, dtype=np.int64)


def attribution_oracle(pages, k, shard_len, geom, records):
    """(per-record [mask, damaged, uncorrectable], unowned) of flagged pages."""
    offs, ends, order = spans(records)
    n = len(records)
    cnt = np.zeros((2, n + 1), dtype=np.int64)    # column n: unowned
    mask = np.zeros(n, dtype=np.int64)
    for g, bm, unc in pages:
        x = np.arange(g * PAGE, min((g + 1) * PAGE, shard_len), dtype=np.int64)
        for i in range(k) if unc else [i for i in range(k) if bm >> i & 1]:
            d = dat_offsets(k, i, x, **geom)
            p = np.searchsorted(offs, d, side="right") - 1
            ok = (d >= 0) & (p >= 0)
            ok[ok] &= d[ok] < ends[p[ok]]
            own = np.where(ok, p, n)
            np.add.at(cnt[int(unc)], own, 1)
            mask[np.unique(own[own < n])] |= 1 << i
    per = [[0, 0, 0] for _ in range(n)]
    for s in range(n):
        per[order[s]] = [int(mask[s]), int(cnt[0, s]), int(cnt[1, s])]
    return per, [int(cnt[0, n]), int(cnt[1, n])]


def attribution_loop(pages, k, shard_len, walk, records):
    """The definition, one byte at a time: the blocks encodeDatFile lays down, and the bisect owner."""
    owner = Owners(records)
    per = [[0, 0, 0] for _ in records]
    unowned = [0, 0]
    for g, bm, unc in pages:
        for i in range(k):
            if not (unc or bm >> i & 1):
                continue
            for x in range(g * PAGE, min((g + 1) * PAGE, shard_len)):
                j = owner(walk(i, x))
                if j < 0:
                    unowned[int(unc)] += 1
                else:
                    per[j][0] |= 1 << i
                    per[j][2 if unc else 1] += 1
    return per, unowned


def invariants(pages, k, shard_len, per, unowned):
    plen = [min(PAGE, shard_len - g * PAGE) for g, _, _ in pages]
    assert sum(p[1] for p in per) + unowned[0] == sum(bin(bm & ((1 << k) - 1)).count("1") * n
                                                    for (_, bm, unc), n in zip(pages, plen) if not unc)
    assert sum(p[2] for p in per) + unowned[1] == k * sum(n for (_, _, unc), n in zip(pages, plen) if unc)


def odd_records(rng, live, dat_size):
    """live, plus records a corrupt .ecx can hold: one overlapping its neighbour, one tied with another's offset, one of
    negative size, one reaching past the end of the .dat."""
    extra = [(900_001, live[3][1] + 5, 4000), (900_002, live[7][1], 10), (900_003, live[9][1], -1),
             (900_004, dat_size - 50, 5000), (900_005, live[-1][1] + 3, 30)]
    recs = list(live) + extra
    rng.shuffle(recs)
    return recs


def random_pages(rng, n_pages, k, m, density, every=False):
    pages = []
    for g in range(n_pages):
        if not every and rng.random() >= density:
            continue
        if rng.random() < 0.3:
            pages.append((g, 0, True))
        else:
            ids = rng.choice(k + m, size=int(rng.integers(1, 3)), replace=False)
            pages.append((g, int(sum(1 << int(i) for i in ids)), False))
    return pages


# ---------------------------------------------------------------------------------------------- CPU

TINY = [(3, 10000, 100, 3 * 10000 + 47 * 300 + 17),       # one large row, small blocks, a zero-padded tail
        (4, 4096 * 3, 512, 2 * 4096 * 3 * 4 + 9 * 512 * 4),  # page-aligned large blocks, a whole tail row
        (5, 7000, 1000, 7000 * 5 + 3000)]                   # a page straddling the large -> small seam


@pytest.mark.parametrize("k,large,small,dat_size", TINY)
def test_oracle_is_the_per_byte_definition(k, large, small, dat_size):
    rng = np.random.default_rng(dat_size)
    _, live = image(rng, dat_size)
    recs = odd_records(rng, live, dat_size)
    shard_len = rn.expected_shard_size(dat_size, k, large, small)
    n_pages = (shard_len + PAGE - 1) // PAGE
    walk = Striping(k, dat_size, large, small)
    geom = encode_geometry(k, dat_size, large, small)
    for i in range(k):      # the vectorised striping is the walk of encodeDatFile's blocks
        x = np.arange(shard_len)
        assert list(dat_offsets(k, i, x, **geom)) == [walk(i, int(v)) for v in x]
    for pages in (random_pages(rng, n_pages, k, 2, 0.5), random_pages(rng, n_pages, k, 2, 1, every=True)):
        want = attribution_loop(pages, k, shard_len, walk, recs)
        assert attribution_oracle(pages, k, shard_len, geom, recs) == want
        invariants(pages, k, shard_len, *want)
        assert any(p[1] or p[2] for p in want[0])
    assert want[1] != [0, 0]                     # every page flagged: the superblock, gaps and padding are unowned


def raw_records_call(swec, device=-1, k=10, m=4, shard_len=None, dat_size=1_000_000, large=10000, small=100,
                     pages=((0, 1, 0),), n_pages=None, records=((1, 8, 100),), n_records=None, unowned=True):
    from seaweedfs_b200._native import NeedleDamage, SketchPage
    L = swec.lib()
    if shard_len is None:
        shard_len = rn.expected_shard_size(dat_size, k, large, small) if k > 0 and large > 0 and small > 0 else 0
    parr = None
    if pages is not None:
        parr = (SketchPage * max(1, len(pages)))()
        for a, (g, bm, unc) in zip(parr, pages):
            a.page, a.blamed_mask, a.uncorrectable = g, bm, unc
    rarr = None
    if records is not None:
        rarr = (NeedleDamage * max(1, len(records)))()
        for r, (nid, off, size) in zip(rarr, records):
            r.needle_id, r.offset, r.size = nid, off, size
            r.damaged_bytes = 77
    un = (C.c_uint64 * 2)(5, 5) if unowned else None
    rc = L.swec_sketch_needle_damage(device, k, m, shard_len, dat_size, large, small, parr,
                                     len(pages or ()) if n_pages is None else n_pages, rarr,
                                     len(records or ()) if n_records is None else n_records, un)
    return rc, L.swec_last_error(), rarr, un


def test_records_call_argument_rules_and_order(swec):
    def status(**kw):
        rc, err, _, _ = raw_records_call(swec, **kw)
        return rc, err

    assert status(k=0)[0] == -1 and b"data_shards" in status(k=0)[1]
    assert status(m=0)[0] == -1 and status(k=20, m=13)[0] == -1
    assert status(k=0, pages=None)[1] == status(k=0)[1]                      # the ratio first
    assert status(large=0, shard_len=5)[0] == -1 and b"geometry" in status(large=0, shard_len=5)[1]
    assert status(dat_size=-1, shard_len=0)[0] == -1
    assert status(shard_len=12345)[0] == -1 and b"shard_len" in status(shard_len=12345)[1]
    assert b"shard_len" in status(shard_len=12345, pages=None)[1]            # before the pages
    assert status(n_pages=-1)[0] == -1 and b"n_pages" in status(n_pages=-1)[1]
    assert b"n_pages" in status(pages=None, n_pages=1)[1]
    assert b"n_pages" in status(pages=None, n_pages=1, unowned=False)[1]     # before the records rules
    assert status(unowned=False)[0] == -1 and b"unowned" in status(unowned=False)[1]
    assert b"records" in status(records=None, n_records=2)[1]
    assert b"unowned" in status(unowned=False, pages=((5, 1, 0), (5, 1, 0)))[1]   # before the page contents
    for bad, what in [(((3, 1, 0), (3, 2, 0)), b"ascending"), (((4, 1, 0), (3, 2, 0)), b"ascending"),
                      (((-1, 1, 0),), b"ascending"), (((10_000, 1, 0),), b"ascending"),
                      (((0, 1, 2),), b"uncorrectable must be 0 or 1"), (((0, 1, 1),), b"mask 0"),
                      (((0, 0, 0),), b"non-zero mask"), (((0, 1 << 14, 0),), b"non-zero mask")]:
        rc, err = status(pages=bad)
        assert rc == -1 and what in err and b"pages[" in err, (bad, err)
    n_pages = (rn.expected_shard_size(1_000_000, 10, 10000, 100) + PAGE - 1) // PAGE
    assert status(pages=((n_pages - 1, 1 << 13, 0),))[0] == -7               # last page, last parity shard: valid
    assert status(pages=((n_pages, 1, 0),))[0] == -1
    assert status(k=20, m=12, pages=((0, 0x80000000, 0),))[0] == -7          # 32 shards: every mask bit is a shard
    assert status()[0] == -7                                                 # every rule passed: no device
    # no pages: zero counts and no GPU work, even for device < 0
    rc, _, rarr, un = raw_records_call(swec, pages=(), records=((1, 8, 100), (2, 200, 50)))
    assert rc == 0 and list(un) == [0, 0] and all(r.damaged_bytes == r.uncorrectable_bytes == r.shard_mask == 0
                                                   for r in rarr)
    assert raw_records_call(swec, pages=None, n_pages=0, records=None)[0] == 0


def cpu_handle(tmp_path, name="5", drop=()):
    from test_needle_damage import cpu_volume
    base = cpu_volume(tmp_path, name=name)
    for i in drop:
        os.remove(base + ".ec%02d" % i)
    return base


def raw_handle_sketch(swec, vol, shard_len=None, pages=((0, 1, 0),), n_pages=None, needles_cap=4, needles=True,
                      n_needles=True, unowned=True, h=True):
    from seaweedfs_b200._native import NeedleDamage, SketchPage
    L = swec.lib()
    if shard_len is None:
        shard_len = os.path.getsize(vol._base + ".ec00")
    parr = None
    if pages is not None:
        parr = (SketchPage * max(1, len(pages)))()
        for a, (g, bm, unc) in zip(parr, pages):
            a.page, a.blamed_mask, a.uncorrectable = g, bm, unc
    arr = (NeedleDamage * max(1, needles_cap))() if needles else None
    nn, un = C.c_int(-5), (C.c_uint64 * 2)(5, 5) if unowned else None
    rc = L.swec_ec_volume_sketch_needle_damage(vol._h if h else None, shard_len, parr,
                                               len(pages or ()) if n_pages is None else n_pages, arr, needles_cap,
                                               C.byref(nn) if n_needles else None, un)
    return rc, L.swec_last_error(), nn.value, un


def test_handle_sketch_needle_damage_rules_and_order(swec, tmp_path):
    ec = swec.erasure_coding
    base = cpu_handle(tmp_path)
    vol = ec.EcVolume(base, device=-1)
    vol._base = base

    def status(**kw):
        return raw_handle_sketch(swec, vol, **kw)[:2]

    assert status(needles_cap=-1)[0] == -1 and b"needles_cap" in status(needles_cap=-1)[1]
    assert b"needles_cap" in status(needles=False)[1]
    assert b"unowned" in status(unowned=False)[1]
    assert b"needles_cap" in status(needles_cap=-1, h=False)[1]              # the needle rules first
    assert status(h=False)[0] == -1 and b"NULL" in status(h=False)[1]
    assert status(n_needles=False)[0] == -1
    assert b"shard_len" in status(shard_len=-1)[1]
    assert b"n_pages" in status(n_pages=-1)[1] and b"n_pages" in status(pages=None, n_pages=2)[1]
    assert b"ascending" in status(pages=((1, 1, 0), (1, 2, 0)))[1]
    assert b"mask" in status(pages=((0, 1 << 14, 0),))[1]
    assert b"ascending" in status(pages=((0, 1, 0),), shard_len=0)[1]
    assert b"ascending" in status(pages=((0, 1, 0), (0, 1, 0)), shard_len=12345)[1]   # the arguments before the files
    rc, err = status(shard_len=12345)
    assert rc == -6                                                          # a local shard of another length
    rc, _, nn, un = raw_handle_sketch(swec, vol, shard_len=12345, pages=())
    assert rc == -6
    rc, _, nn, un = raw_handle_sketch(swec, vol, pages=())
    assert rc == 0 and nn == 0 and list(un) == [0, 0]                        # no pages: no GPU work
    assert status()[0] == -7                                                 # every check passed: no device
    vol.close()


def raw_page_sketch(swec, vol, want, cap=4, null=(), total=14):
    L = swec.lib()
    bufs = {i: np.zeros(max(cap, 1), dtype=np.uint64) for i in want}
    ptrs = (C.c_void_p * total)(*[bufs[i].ctypes.data if i in bufs else None for i in range(total)])
    sl, n = C.c_int64(-1), C.c_int64(-1)
    rc = L.swec_ec_volume_page_sketch(None if "vol" in null else vol._h, 1, None if "sketches" in null else ptrs, cap,
                                      None if "len" in null else C.byref(sl), None if "n" in null else C.byref(n))
    return rc, L.swec_last_error(), sl.value, n.value


def test_handle_page_sketch_rules_and_order(swec, tmp_path):
    ec = swec.erasure_coding
    base = cpu_handle(tmp_path, drop=(4,))
    vol = ec.EcVolume(base, device=-1)
    for null in ("vol", "sketches", "len", "n"):
        assert raw_page_sketch(swec, vol, [0], null=(null,))[0] == -1
    rc, err, _, _ = raw_page_sketch(swec, vol, [0], cap=-1)
    assert rc == -1 and b"sketches_cap" in err
    rc, err, _, _ = raw_page_sketch(swec, vol, [])
    assert rc == -1 and b"no shard requested" in err
    rc, err, _, _ = raw_page_sketch(swec, vol, [0, 4], cap=-1)
    assert rc == -1                                                          # the arguments before the shards
    rc, err, _, _ = raw_page_sketch(swec, vol, [0, 4])
    assert rc == -2 and b".ec04" in err
    with open(base + ".ec07", "r+b") as f:
        f.truncate(os.path.getsize(base + ".ec07") - 1)
    vol.close()
    vol = ec.EcVolume(base, device=-1)
    assert raw_page_sketch(swec, vol, [3, 4, 7])[0] == -2                    # not local before unequal lengths
    assert raw_page_sketch(swec, vol, [3, 7])[0] == -6
    assert raw_page_sketch(swec, vol, [3, 8])[0] == -7                       # every check passed: no device
    assert raw_page_sketch(swec, vol, [7])[0] == -7
    vol.close()
    # empty shards: no pages and no GPU work, even for device < 0
    for i in range(14):
        if os.path.exists(base + ".ec%02d" % i):
            open(base + ".ec%02d" % i, "wb").close()
    vol = ec.EcVolume(base, device=-1)
    rc, _, sl, n = raw_page_sketch(swec, vol, [0, 13])
    assert (rc, sl, n) == (0, 0, 0)
    vol.close()


def test_new_entry_points_are_bound(swec):
    from seaweedfs_b200 import _native
    for name in ("swec_sketch_needle_damage", "swec_ec_volume_sketch_needle_damage", "swec_ec_volume_page_sketch"):
        assert name in _native.PROTOTYPES and getattr(swec.lib(), name)


# ---------------------------------------------------------------------------------------------- GPU: records level


def device_call(swec, pages, k, m, shard_len, dat_size, large, small, records):
    res = swec.erasure_coding.sketch_needle_damage(pages, shard_len, dat_size, records, k, m, large, small)
    assert [(r["needle_id"], r["offset"], r["size"]) for r in res["needles"]] == [tuple(r) for r in records]
    return [[r["shard_mask"], r["damaged_bytes"], r["uncorrectable_bytes"]] for r in res["needles"]], res["unowned"]


GRID = [(10, 4, 10000, 100, 2 * 10000 * 10 + 37 * 100 * 10 + 450),
        (10, 4, 4096, 512, 3 * 4096 * 10 + 11 * 512 * 10 + 99),
        (6, 3, 3000, 1000, 2 * 3000 * 6 + 5 * 1000 * 6 + 1),
        (20, 12, 8192, 4096, 8192 * 20 * 2 + 4096 * 20 * 3),
        (20, 12, 10000, 100, 10000 * 20 + 100 * 20 * 13 + 1234)]


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,large,small,dat_size", GRID)
def test_records_call_is_the_oracle(cuda, swec, k, m, large, small, dat_size):
    rng = np.random.default_rng(dat_size + k)
    _, live = image(rng, dat_size)
    recs = odd_records(rng, live, dat_size)
    shard_len = rn.expected_shard_size(dat_size, k, large, small)
    n_pages = (shard_len + PAGE - 1) // PAGE
    geom = encode_geometry(k, dat_size, large, small)
    for pages in (random_pages(rng, n_pages, k, m, 0.3), random_pages(rng, n_pages, k, m, 1, every=True),
                  [(n_pages - 1, 1 << (k - 1), False)], [(0, 0, True)]):
        want = attribution_oracle(pages, k, shard_len, geom, recs)
        assert device_call(swec, pages, k, m, shard_len, dat_size, large, small, recs) == want
        invariants(pages, k, shard_len, *want)


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", [(10, 4), (6, 3)])
def test_records_call_on_pages_of_the_checked_locate(cuda, swec, k, m):
    """Pages located from real sketches of a set with lost shards: damage in whole pages of data shards."""
    large, small = 10000, 100
    dat_size = 2 * large * k + 60 * small * k + 321
    rng = np.random.default_rng(k * 7)
    dat, live = image(rng, dat_size)
    shards = rn.encode_dat_image(dat, k, m, large, small)
    shard_len = len(shards[0])
    n_pages = (shard_len + PAGE - 1) // PAGE
    for g in range(n_pages):
        for i in rng.choice(k, size=int(rng.integers(0, 3)), replace=False):
            shards[int(i)][g * PAGE:(g + 1) * PAGE] ^= np.uint8(0x3C)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    sk = _device_sketches(cuda, enc, shards, 0xC0FFEE)
    sk[k + 1] = None                                                          # a lost parity shard: c = m - 1
    res = enc.locate_sketch_damage_checked(sk, shard_len, radius=1)
    enc.close()
    pages = res["pages"]
    assert any(not p[2] for p in pages)
    want = attribution_oracle(pages, k, shard_len, encode_geometry(k, dat_size, large, small), live)
    assert device_call(swec, pages, k, m, shard_len, dat_size, large, small, live) == want
    invariants(pages, k, shard_len, *want)


def held_before(d, i, k, large, small, large_rows):
    """How many bytes of the .dat range [0, d) data shard i holds (encode geometry, d within the .dat)."""
    d = np.asarray(d, dtype=np.int64)
    lb = large_rows * large * k

    def rows(e, blk):
        return (e // (blk * k)) * blk + np.clip(e % (blk * k) - i * blk, 0, blk)
    return np.where(d <= lb, rows(np.minimum(d, lb), large), large_rows * large + rows(np.maximum(d - lb, 0), small))


@pytest.mark.gpu
def test_records_call_at_full_size(cuda, swec):
    """A 30 GiB volume of ~1 M records: every page of one data shard flagged (786,432 pages), then 64 random pages."""
    k, m, large, small = 10, 4, GIB, MIB
    dat_size = 30 * GIB
    shard_len = rn.expected_shard_size(dat_size, k, large, small)
    n_pages = (shard_len + PAGE - 1) // PAGE
    assert n_pages == 786_432
    rng = np.random.default_rng(30)
    sizes = rng.integers(0, 60_000, 1_100_000)
    actual = 16 + sizes + 4 + 8
    actual += 8 - actual % 8
    gaps = np.where(rng.random(len(sizes)) < 0.05, 8 * rng.integers(1, 64, len(sizes)), 0)
    offs = 8 + np.concatenate([[0], np.cumsum(actual + gaps)[:-1]])
    keep = offs + actual <= dat_size
    offs, sizes, actual = offs[keep], sizes[keep], actual[keep]
    assert 900_000 < len(offs) < 1_100_000
    records = list(zip(range(1, len(offs) + 1), offs.tolist(), sizes.tolist()))
    shard = 3
    pages = [(g, 1 << shard, False) for g in range(n_pages)]
    got, unowned = device_call(swec, pages, k, m, shard_len, dat_size, large, small, records)
    held = held_before(offs + actual, shard, k, large, small, dat_size // (large * k)) - \
        held_before(offs, shard, k, large, small, dat_size // (large * k))
    assert [g[1] for g in got] == held.tolist()
    assert all(g[2] == 0 and g[0] == (1 << shard if h else 0) for g, h in zip(got, held.tolist()))
    assert unowned[1] == 0 and sum(held.tolist()) + unowned[0] == shard_len
    picked = sorted(rng.choice(n_pages, 64, replace=False).tolist())
    pages = [(g, 0, True) if j % 3 == 0 else (g, int(rng.integers(1, 1 << (k + m))), False) for j, g in enumerate(picked)]
    want = attribution_oracle(pages, k, shard_len, encode_geometry(k, dat_size, large, small), records)
    assert device_call(swec, pages, k, m, shard_len, dat_size, large, small, records) == want
    assert any(w[1] for w in want[0]) and any(w[2] for w in want[0])


# ---------------------------------------------------------------------------------------------- GPU: mounted volume


def xor_pages(base, hits, n):
    """XOR 0x5A into every byte of page g of shard i, for (g, i) in hits."""
    for g, i in hits:
        path = base + ".ec%02d" % i
        with open(path, "r+b") as f:
            f.seek(g * PAGE)
            b = np.frombuffer(f.read(min(PAGE, n - g * PAGE)), dtype=np.uint8) ^ np.uint8(0x5A)
            f.seek(g * PAGE)
            f.write(b.tobytes())


@pytest.mark.gpu
@pytest.mark.parametrize("per_page", [1, 2])
def test_handle_equals_the_byte_level_call(cuda, swec, tmp_path, per_page):
    """Whole pages XORed, one data shard per page (blamed at radius 1) or two (uncorrectable): the sketch path from
    page_sketch to sketch_needle_damage names exactly what swec_ec_volume_locate_needle_damage names."""
    ec = swec.erasure_coding
    base, _, _ = generated_volume(swec, tmp_path, "3", dat_size=5_000_000)
    n = os.path.getsize(base + ".ec00")
    n_pages = (n + PAGE - 1) // PAGE
    rng = np.random.default_rng(per_page)
    hits = []
    for g in sorted(rng.choice(n_pages - 1, 12, replace=False).tolist()) + [n_pages - 1]:
        hits += [(g, int(i)) for i in rng.choice(10, per_page, replace=False)]
    xor_pages(base, hits, n)
    vol = ec.EcVolume(base)
    sk, shard_len = vol.page_sketch(0x5EED + per_page)
    assert shard_len == n and sorted(sk) == list(range(14))
    enc = ec.Encoder(10, 4)
    loc = enc.locate_sketch_damage([sk[i] for i in range(14)], shard_len, radius=1)
    enc.close()
    assert [p[0] for p in loc["pages"]] == sorted({g for g, _ in hits})
    assert all(p[2] == (per_page == 2) for p in loc["pages"])
    got = vol.sketch_needle_damage(loc["pages"], shard_len)
    want = vol.locate_needle_damage(radius=1)
    assert got["n_needles"] == want["n_needles"] > 0
    assert got["needles"] == want["needles"] and got["unowned"] == want["unowned"]
    assert sum(r["uncorrectable_bytes" if per_page == 2 else "damaged_bytes"] for r in got["needles"]) > 0
    vol.close()


@pytest.mark.gpu
def test_handle_with_some_shards_elsewhere(cuda, swec, tmp_path):
    """Attribution needs no local shard bytes: a handle with 3 local shards (others in another directory or gone), and
    one with none of the flagged shards, name the same needles as the handle of the whole set."""
    ec = swec.erasure_coding
    base, _, _ = generated_volume(swec, tmp_path, "4", dat_size=4_000_000)
    n = os.path.getsize(base + ".ec00")
    pages = [(0, 1, False), (5, 1 << 3 | 1 << 12, False), (9, 0, True), ((n - 1) // PAGE, 1 << 9, False)]
    full = ec.EcVolume(base)
    want = full.sketch_needle_damage(pages, n)
    full.close()
    assert want["n_needles"] > 0
    other = tmp_path / "elsewhere"
    other.mkdir()
    for i in range(14):
        if i in (2, 11, 13):
            continue
        if i % 2:
            os.remove(base + ".ec%02d" % i)
        else:
            os.rename(base + ".ec%02d" % i, str(other / ("4.ec%02d" % i)))
    part = ec.EcVolume(base)
    assert part.info()["local_shards"] == [2, 11, 13]
    assert part.sketch_needle_damage(pages, n) == want
    with pytest.raises(swec._native.SwecError) as e:
        part.sketch_needle_damage(pages, n + 1)
    assert e.value.status == -6
    part.close()
    for i in (2, 11, 13):
        os.remove(base + ".ec%02d" % i)
    open(base + ".ec02", "wb").write(b"x" * n)             # one local shard of the right length
    alone = ec.EcVolume(base)
    assert alone.sketch_needle_damage(pages, n) == want
    alone.close()


@pytest.mark.gpu
def test_handle_page_sketch_is_the_file_sketch(cuda, swec, tmp_path):
    """Every local shard, a subset, a subset of a handle with shards elsewhere, ragged lengths and a cap below the page
    count: the words of page_sketch_file, bit for bit."""
    ec = swec.erasure_coding
    base, dirs, files = _generate(swec, tmp_path, 10, 4, seed=9)      # 90,000-byte shards: the last page is partial
    open(base + ".ecx", "wb").close()
    n = os.path.getsize(files[0])
    assert n % PAGE
    vol = ec.EcVolume(base, additional_dirs=dirs)
    seed = 0xFEED
    want = {i: ec.page_sketch_file(files[i], seed)[0] for i in range(14)}
    sk, shard_len = vol.page_sketch(seed)
    assert shard_len == n and sorted(sk) == list(range(14))
    assert all(np.array_equal(sk[i], want[i]) for i in range(14))
    sk, _ = vol.page_sketch(seed, shards=[13, 0, 6])
    assert sorted(sk) == [0, 6, 13] and all(np.array_equal(sk[i], want[i]) for i in sk)
    L = swec.lib()
    cap = 5
    bufs = {i: np.full(cap + 2, 7, dtype=np.uint64) for i in (1, 12)}
    ptrs = (C.c_void_p * 14)(*[bufs[i].ctypes.data if i in bufs else None for i in range(14)])
    sl, npg = C.c_int64(0), C.c_int64(0)
    assert L.swec_ec_volume_page_sketch(vol._h, seed, ptrs, cap, C.byref(sl), C.byref(npg)) == 0
    assert (sl.value, npg.value) == (n, (n + PAGE - 1) // PAGE) and npg.value > cap
    assert all(np.array_equal(bufs[i][:cap], want[i][:cap]) and (bufs[i][cap:] == 7).all() for i in bufs)
    vol.close()
    part = ec.EcVolume(base, additional_dirs=[dirs[i] for i in (2, 5, 11)])
    assert part.info()["local_shards"] == [2, 5, 11]
    sk, _ = part.page_sketch(seed)
    assert sorted(sk) == [2, 5, 11] and all(np.array_equal(sk[i], want[i]) for i in sk)
    part.close()
    for size in (1, PAGE, PAGE + 1, 3 * PAGE - 1):                      # ragged lengths, shared by the set
        for f in files:
            os.truncate(f, size)
        vol = ec.EcVolume(base, additional_dirs=dirs)
        sk, shard_len = vol.page_sketch(seed + size, shards=[0, 9, 13])
        assert shard_len == size
        assert all(np.array_equal(sk[i], ec.page_sketch_file(files[i], seed + size)[0]) for i in sk)
        vol.close()
