"""The locate kernel's bookkeeping at every seam: the report and the page runs of swec_locate_kernel (damage.cu) and
DamageLocator::collect, and what the repairs read and write from those runs.

Each lane keeps two runs and flushes one to make room for a third set; a warp merges equal runs and flags the pages of
each set's first and last column; collect walks one page bitmap per set, skipping 32 pages on a zero word, and clips the
last range to the shard.  Pass 2 of the repairs re-reads only the flagged pages (submit_flagged, ec_files.cc) and writes
back only each blamed shard's own pages (PageWrites).  The placement corpus below puts damage on both sides of every seam
of that bookkeeping: the 16-byte vector, the 512-byte warp window, the 4 KiB page, the 32-page bitmap word, the partial
last vector and the clipped last page; three and four sets in one lane's columns and in every lane of a warp; one set's
columns on both sides of a page inside one warp window (file level, where item bases are 256 bytes off a window); runs
of 1, 2, 31, 32 and 33 pages, two shards' runs touching page by page, and uncorrectable columns inside blamed runs.

Expected values come from the existing oracles only: damage_oracle.decode_columns / report (blame, report, page runs),
the checked rebuild and decode oracles of test_checked_rebuild.py / test_checked_decode.py, test_damage_repair.correct
(repaired bytes) and the needle walks of test_needle_damage.py.  Every call is compared field by field.

cpu: the corpus reaches both sides of every seam class; a restatement of submit_flagged / PageWrites on hand-made runs;
the swec_locate_kernel symbols of libswec.so are exactly the nine the GPU part runs.
gpu: every instantiation of the locate kernel through the four device calls, aligned and on the byte path, over the
corpus at eleven shard lengths, with max_ranges 0, 1 and n_ranges - 1 and across the 256 MiB piece boundary, the
instantiation of each configuration confirmed by torch.profiler in a child process; locate_ec_damage and
repair_ec_damage at item sizes 256, 768, 4096, 4352 and 65536 (the pass-2 item count from SWEC_PIPE_STATS); the mounted
volume's locate_needle_damage / repair_needle_damage on records that start and end on page and item seams; O_DIRECT.
"""
from __future__ import annotations

import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import damage_oracle as do  # noqa: E402
import needle_oracle as no  # noqa: E402
import test_checked_decode as tcd  # noqa: E402
import test_checked_rebuild as tcr  # noqa: E402
import test_damage_exhaustive as tde  # noqa: E402
import test_damage_repair as tdr  # noqa: E402
import test_decode_exhaustive as tdx  # noqa: E402
import test_kernel_variants as tkv  # noqa: E402
import test_needle_damage as tnd  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGE = 4096
WORD = 32 * PAGE                   # the columns of one 32-bit word of a page bitmap
WINDOW = 512                       # the columns of one warp's turn: 32 lanes x 16 bytes
PIECE = 256 << 20                  # device calls launch the locate kernel on pieces of this many columns
LENGTHS = [1, 15, 16, 17, 512, 4095, 4096, 4097, WORD - 1, WORD + 1, 65 * PAGE + 5]
FILE_LEN = 65 * PAGE + 5
FILE_CHUNKS = [256, 768, 4096, 4352, 65536]
PAST_NS = tdr.PAST_NS
LOCATE, CORRECT, REBUILD, DECODE = tdx.LOCATE, tdx.CORRECT, tdx.REBUILD, tdx.DECODE

# (call, k, m, lost, radius, the (MT, MODE) instantiation of swec_locate_kernel it runs)
ROUTES = [("locate", 10, 4, (), 1, (4, LOCATE)), ("locate", 10, 4, (), 2, (4, LOCATE)),
          ("locate", 6, 3, (), 1, (0, LOCATE)), ("locate", 20, 12, (), 1, (0, LOCATE)),
          ("locate", 3, 2, (), 1, (0, LOCATE)),
          ("correct", 10, 4, (), 1, (4, CORRECT)), ("correct", 10, 4, (), 2, (4, CORRECT)),
          ("correct", 6, 3, (), 1, (0, CORRECT)), ("correct", 20, 12, (), 1, (0, CORRECT)),
          ("correct", 3, 2, (), 1, (0, CORRECT)),
          ("rebuild", 10, 4, (3,), 1, (3, REBUILD)), ("rebuild", 10, 4, (12,), 1, (3, REBUILD)),
          ("rebuild", 10, 4, (2, 7), 1, (0, REBUILD)), ("rebuild", 10, 4, (), 2, (0, REBUILD)),
          ("rebuild", 6, 3, (1,), 1, (0, REBUILD)),
          ("decode", 10, 4, (), 2, (4, DECODE)), ("decode", 10, 4, (3,), 1, (3, DECODE)),
          ("decode", 10, 4, (12,), 1, (3, DECODE)), ("decode", 10, 4, (2, 7), 1, (0, DECODE)),
          ("decode", 6, 3, (1,), 1, (0, DECODE))]


def route_id(r):
    call, k, m, lost, radius, _ = r
    return "%s-rs%d.%d-lost%s-r%d" % (call, k, m, "_".join(map(str, lost)) or "0", radius)


# ---------------------------------------------------------------------------------------------- placement corpus


def roles(k, m, lost=()):
    """Distinct present shards for the roles of a placement: two data shards, a first and a last parity shard, and a
    fourth blamed shard."""
    present = [i for i in range(k + m) if i not in lost]
    data = [i for i in present if i < k]
    return {"A": data[0], "B": data[-1], "P": next(i for i in present if i >= k), "P2": present[-1],
            "X": present[1]}


def corpus(n, k, m, radius, lost=()):
    """name -> one damage placement on shards of n columns: a sorted list of (column, shard ids).  A column wrong in
    radius + 1 shards (U) is beyond the radius; what the decoder makes of it is the oracle's to say."""
    r = roles(k, m, lost)
    A, B, P, P2, X = r["A"], r["B"], r["P"], r["P2"], r["X"]
    present = [i for i in range(k + m) if i not in lost]
    U = tuple(sorted({A, B, P2} if radius >= 2 else {A, B}))[:radius + 1]
    if len(U) < radius + 1:
        U = tuple(present[:radius + 1])
    rot = [(A,), (P,), (B,), (X,), (P2,)]
    out = {}

    seams = [0, 15, 16, 17, 511, 512, 513, PAGE - 1, PAGE]
    seams += [p * PAGE + q for p in (31, 32, 33, 63, 64, 65) for q in (0, PAGE - 1)]
    seams += [n - 1]
    if n % 16:
        seams += [n - n % 16 - 1, n - n % 16]              # the last whole vector, then the partial one
    if n % PAGE:
        seams += [n - n % PAGE - 1, n - n % PAGE + (n % PAGE) // 2]   # the page before the clipped one, and inside it
    cols = sorted({c for c in seams if 0 <= c < n})
    out["seams"] = [(c, rot[j % len(rot)]) for j, c in enumerate(cols)]

    lane = [(A,), (B,), (P,), U, (X,), (A,), (B,), (P,), (X,), U, (P,), (A,)]    # sets 3 and 4 flush run[1]
    v = 5 * PAGE // 16 + 7
    out["lane mix"] = [(v * 16 + c, s) for c, s in enumerate(lane)]
    w = 7 * PAGE                                           # one warp window, every lane with the mix rotated
    out["warp mix"] = [(w + 16 * ln + c, lane[(c + ln) % len(lane)]) for ln in range(32) for c in range(len(lane))]

    # one set's columns either side of a page boundary: inside one warp window at item sizes 768 (boundary 1 and 4)
    # and 4352 (boundaries 2 and 4)
    out["straddle"] = [(b * PAGE + d, s) for b, s in ((1, (A,)), (2, (P,)), (4, (B,))) for d in (-6, 4)]

    last = (n - 1) // PAGE
    runs = []
    for s, first, pages, at in ((A, 64, 1, 100), (B, 3, 2, 200), (P, 1, 31, 300), (X, 0, 32, 400),
                                (P2, last - 32, 33, 500)):
        runs += [(p * PAGE + (at if p < last else min(at, (n - 1) % PAGE)), (s,))
                 for p in range(max(first, 0), first + pages)]
    out["runs"] = runs
    out["interleave"] = [(p * PAGE + 2048, (A,) if p % 2 else (B,)) for p in range(40, 48)]
    out["unc in runs"] = ([(p * PAGE + 300, (A,)) for p in range(8, 14)] + [(p * PAGE + 400, (P,)) for p in range(10, 16)]
                          + [(p * PAGE + 500, U) for p in range(9, 12)] + [(15 * PAGE + 4095, U), (16 * PAGE, (A,))])
    cases = {}
    for name, pl in out.items():
        first = {}
        for c, s in pl:                       # on short shards the runs' last page can land on one column: first wins
            if 0 <= c < n:
                first.setdefault(c, tuple(s))
        pl = sorted(first.items())
        if pl and pl not in cases.values():
            cases[name] = pl
    return cases


def apply(shards, placement, seed):
    """The shards with a random non-zero byte XORed into every (column, shard) of the placement."""
    rng = np.random.default_rng(seed)
    out = [None if s is None else s.copy() for s in shards]
    for c, ids in placement:
        for s in ids:
            out[s][c] ^= np.uint8(rng.integers(1, 256))
    return out


def page_runs(cols):
    """Maximal runs of pages holding a column: [(first page, pages)]"""
    pages = sorted({c // PAGE for c in cols})
    runs = []
    for p in pages:
        if runs and runs[-1][0] + runs[-1][1] == p:
            runs[-1][1] += 1
        else:
            runs.append([p, 1])
    return [tuple(r) for r in runs]


def straddles(lo, hi, chunk):
    """Whether columns lo < hi lie on two pages inside one warp window of a pipeline item of `chunk` columns."""
    base = lo // chunk * chunk
    win = base + (lo - base) // WINDOW * WINDOW
    return hi // chunk * chunk == base and hi < win + WINDOW and lo // PAGE != hi // PAGE


def seam_classes(n, cases):
    """Which side of which seam class the placements of shards of n columns reach."""
    got = set()
    for pl in cases.values():
        cols = {c for c, _ in pl}
        per = {}
        for c, ids in pl:
            per.setdefault(ids if len(ids) == 1 else "U", []).append(c)
        for edge, name in ((16, "vector"), (WINDOW, "window"), (PAGE, "page"), (WORD, "bitmap word")):
            for c in cols:
                if c % edge == edge - 1 and c + 1 in cols:
                    got.add(name + " both sides")
            if any(c % edge == 0 and c - 1 not in cols for c in cols if c):
                got.add(name + " first column alone")
        for key, cs in per.items():           # a set's first page of a word flagged after a zero word of its own
            pages = {c // PAGE for c in cs}
            if any(p % 32 == 0 and p - 1 not in pages and not pages & set(range(p - 32, p)) for p in pages if p):
                got.add("bitmap word first page after a zero word")
        for w in (31, 63):
            if {w, w + 1} <= {c // PAGE for c in cols}:
                got.add("pages %d/%d" % (w, w + 1))
        if n % 16 and any(c >= n - n % 16 for c in cols) and n - n % 16 - 1 in cols:
            got.add("partial last vector")
        if n % PAGE and any(c >= n - n % PAGE for c in cols) and any(n - n % PAGE - PAGE <= c < n - n % PAGE for c in cols):
            got.add("clipped last page")
        if n - 1 in cols:
            got.add("last column")
        vec = {}
        for c, ids in pl:
            vec.setdefault(c // 16, set()).add(ids)
        if any(len(s) >= 4 for s in vec.values()):
            got.add("four sets in one lane")
        for wb in {c // WINDOW for c in cols}:
            if all(len(vec.get(wb * 32 + ln, ())) >= 3 for ln in range(32)):
                got.add("three sets in every lane of a warp")
        for key, cs in per.items():
            for lo in cs:
                for hi in cs:
                    if lo < hi:
                        for chunk in (768, 4352):
                            if key != "U" and straddles(lo, hi, chunk):
                                got.add("straddle at %d" % chunk)
            for _, pages in page_runs(cs):
                if key != "U" and pages in (1, 2, 31, 32, 33):
                    got.add("run of %d pages" % pages)
        runs = {key: page_runs(cs) for key, cs in per.items() if key != "U"}
        for a in runs:
            for b in runs:
                if a != b and any(p + q == r for p, q in runs[a] for r, _ in runs[b]):
                    got.add("touching runs of two shards")
        blamed = {c // PAGE for key, cs in per.items() if key != "U" for c in cs}
        if any(c // PAGE in blamed for c in per.get("U", [])):
            got.add("uncorrectable inside a blamed run")
    return got


SEAM_CLASSES = {"vector both sides", "window both sides", "page both sides", "bitmap word both sides",
                "vector first column alone", "window first column alone", "page first column alone",
                "bitmap word first page after a zero word", "pages 31/32", "pages 63/64", "partial last vector",
                "clipped last page", "last column", "four sets in one lane", "three sets in every lane of a warp",
                "straddle at 768", "straddle at 4352", "run of 1 pages", "run of 2 pages", "run of 31 pages",
                "run of 32 pages", "run of 33 pages", "touching runs of two shards", "uncorrectable inside a blamed run"}


# ---------------------------------------------------------------------------------------------- expected values


def locate_expected(shards, k, m, radius):
    cols, a, b, va, vb, _ = do.decode_columns(shards, k, m, radius)
    rep = tde.without_ok(do.report(len(shards[0]), k + m, cols, a, b))
    fixed = [s.copy() for s in shards]
    for pos, val in ((a, va), (b, vb)):
        for sid in range(k + m):
            sel = pos == sid
            fixed[sid][cols[sel]] ^= val[sel]
    return rep, fixed


def pass2_items(ranges, chunk):
    """submit_flagged: the page runs sorted and merged into maximal spans, touching ones included, each cut into items of
    at most `chunk` columns: [(offset, length)]."""
    spans = []
    for lo, hi in sorted((o, o + ln) for _, o, ln in ranges):
        if spans and lo <= spans[-1][1]:
            spans[-1][1] = max(spans[-1][1], hi)
        else:
            spans.append([lo, hi])
    return [(o, min(chunk, hi - o)) for lo, hi in spans for o in range(lo, hi, chunk)]


def page_writes(ranges, items):
    """PageWrites: per item, each blamed shard's own pages in it, [(item, shard, offset, length)]."""
    out = []
    for j, (o, ln) in enumerate(items):
        for sid in sorted({s for s, _, _ in ranges if s >= 0}):
            for s, ro, rl in ranges:
                lo, hi = max(ro, o), min(ro + rl, o + ln)
                if s == sid and lo < hi:
                    out.append((j, sid, lo, hi - lo))
    return out


# ---------------------------------------------------------------------------------------------- CPU


def test_corpus_reaches_both_sides_of_every_seam():
    got = set()
    for n in LENGTHS:
        for k, m, radius, lost in ((10, 4, 1, ()), (10, 4, 2, ()), (3, 2, 1, ()), (10, 4, 1, (3,))):
            cases = corpus(n, k, m, radius, lost)
            got |= seam_classes(n, cases)
            for pl in cases.values():           # every role is a present shard, every U column beyond the radius
                assert all(0 <= c < n and not set(ids) & set(lost) for c, ids in pl)
                assert all(len(ids) in (1, radius + 1) for _, ids in pl)
    assert got >= SEAM_CLASSES, sorted(SEAM_CLASSES - got)
    big = seam_classes(FILE_LEN, corpus(FILE_LEN, 10, 4, 1))
    assert big >= SEAM_CLASSES, sorted(SEAM_CLASSES - big)
    assert seam_classes(FILE_LEN, corpus(FILE_LEN, 6, 3, 1)) >= {"straddle at 768", "straddle at 4352",
                                                                   "touching runs of two shards"}


def test_straddles_at_the_item_sizes_that_cut_windows():
    assert straddles(PAGE - 6, PAGE + 4, 768) and not straddles(PAGE - 6, PAGE + 4, 4352)
    assert straddles(2 * PAGE - 6, 2 * PAGE + 4, 4352) and not straddles(2 * PAGE - 6, 2 * PAGE + 4, 768)
    for chunk in (256, 4096, 65536):            # item bases on a window: no window crosses a page
        assert not any(straddles(b * PAGE - 6, b * PAGE + 4, chunk) for b in range(1, 66))


def test_pass2_restatement_on_hand_made_runs():
    # one run longer than several items
    items = pass2_items([(3, 0, 3 * PAGE)], 4352)
    assert items == [(0, 4352), (4352, 4352), (8704, 3584)]
    assert page_writes([(3, 0, 3 * PAGE)], items) == [(0, 3, 0, 4352), (1, 3, 4352, 4352), (2, 3, 8704, 3584)]
    # two shards' runs in one item; touching spans merge, a gap does not
    runs = [(0, 0, PAGE), (5, PAGE, PAGE), (5, 3 * PAGE, PAGE)]
    items = pass2_items(runs, 65536)
    assert items == [(0, 2 * PAGE), (3 * PAGE, PAGE)]
    assert page_writes(runs, items) == [(0, 0, 0, PAGE), (0, 5, PAGE, PAGE), (1, 5, 3 * PAGE, PAGE)]
    assert pass2_items(runs, 768) == [(o, 768) for o in range(0, 7680, 768)] + [(7680, 512)] + \
        [(3 * PAGE + o, min(768, PAGE - o)) for o in range(0, PAGE, 768)]
    # an uncorrectable run overlapping a blamed one: read, never written
    runs = [(2, PAGE, 3 * PAGE), (-1, 2 * PAGE, 4 * PAGE)]
    items = pass2_items(runs, 8192)
    assert items == [(PAGE, 8192), (3 * PAGE, 8192), (5 * PAGE, PAGE)]
    assert page_writes(runs, items) == [(0, 2, PAGE, 8192), (1, 2, 3 * PAGE, PAGE)]
    # a clipped last page: the span ends at the shard's end
    runs = [(1, 64 * PAGE, PAGE + 5), (-1, 65 * PAGE, 5)]
    assert pass2_items(runs, 768)[-1] == (64 * PAGE + 5 * 768, PAGE + 5 - 5 * 768)
    assert sum(ln for _, ln in pass2_items(runs, 768)) == PAGE + 5
    assert page_writes(runs, pass2_items(runs, 768))[-1] == (5, 1, 64 * PAGE + 5 * 768, PAGE + 5 - 5 * 768)


def test_expected_values_for_each_route_on_the_cpu():
    """The expected report of every route's oracle agrees with damage_oracle on a full set (locate, correct), and the
    rebuild and decode oracles blame only present shards."""
    n = 3 * PAGE + 7
    for call, k, m, lost, radius, _ in ROUTES:
        if k + m > 14:
            continue
        clean = tde.random_set(k, m, n, seed=k * 100 + m)
        for name, pl in corpus(n, k, m, radius, lost).items():
            bad = apply(clean, pl, seed=len(pl))
            rep, fixed = locate_expected(bad, k, m, radius)
            if m <= 8:
                assert rep == tde.without_ok(do.locate(bad, k, m, radius)), (call, name)
            if call == "correct" and m <= 8:
                assert tdr.same(fixed, tdr.correct(bad, k, m, radius)), (call, name)
            present = tde.mask(k + m, lost)
            found = [s if present[i] else None for i, s in enumerate(bad)]
            if call == "rebuild":
                _, want = tcr.checked_rebuild(found, k, m, present, radius)
                assert not set(want["shards"]) & set(lost)
            if call == "decode":
                _, want = tcd.checked_decode(found, k, m, present, radius)
                assert not set(want["shards"]) & set(lost)


def test_locate_symbols_are_the_routes(swec):
    """The swec_locate_kernel instantiations in libswec.so are exactly the nine ROUTES reach: a new one fails here
    until a route runs it."""
    from seaweedfs_b200 import _native
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("no CUDA toolkit")
    out = subprocess.run([cuobjdump, "-symbols", _native.library_path()], capture_output=True, text=True,
                         check=True).stdout
    found = {tdx.locate_id(ln.split()[-1]) for ln in out.splitlines() if "STT_FUNC" in ln and "STO_ENTRY" in ln}
    found.discard(None)
    assert found == {r[-1] for r in ROUTES} and len(found) == 9, sorted(found)


# ---------------------------------------------------------------------------------------------- GPU: device level


def upload(torch, shards, shift):
    n = len(shards)
    length = len(next(s for s in shards if s is not None))
    buf = torch.zeros((n, (shift + length + 64 + 255) // 256 * 256), dtype=torch.uint8, device="cuda")
    buf.fill_(0x5A)
    for i, s in enumerate(shards):
        if s is not None:
            buf[i, shift:shift + length] = torch.from_numpy(s).cuda()
    return buf


def rows(buf, shift, length):
    return [buf[i, shift:shift + length].cpu().numpy() for i in range(len(buf))]


def run_route(torch, enc, route, shards, shift, max_ranges=1 << 16):
    """One device call of the route on a copy of `shards` (lost ones None): (result, the shard rows after, before)."""
    call, k, m, lost, radius, _ = route
    length = len(shards[0] if shards[0] is not None else shards[-1])
    buf = upload(torch, shards, shift)
    before = buf.clone()
    p = tde.ptrs(buf, shift)
    present = [int(i not in lost) for i in range(k + m)]
    if call == "locate":
        got = enc.locate_damage_device(p, length, radius=radius, max_ranges=max_ranges)
    elif call == "correct":
        got = enc.correct_damage_device(p, length, radius=radius, max_ranges=max_ranges)
    elif call == "rebuild":
        got = enc.reconstruct_checked_device(p, present, length, radius=radius, max_ranges=max_ranges)
    else:
        for i in lost:
            if i >= k:
                p[i] = None
        got = enc.decode_data_checked_device(p, present, length, radius=radius, max_ranges=max_ranges)
    torch.cuda.synchronize()
    return got, buf, before


def check_route(torch, enc, route, bad, shift):
    """Every field of the report and every byte of every buffer against the route's oracle; returns the report."""
    call, k, m, lost, radius, _ = route
    n = len(bad[0] if bad[0] is not None else bad[-1])
    present = tde.mask(k + m, lost)
    got, buf, before = run_route(torch, enc, route, bad, shift)
    after = rows(buf, shift, n)
    if call in ("locate", "correct"):
        want, fixed = locate_expected(bad, k, m, radius)
        expect = fixed if call == "correct" else bad
    elif call == "rebuild":
        rebuilt, want = tcr.checked_rebuild(bad, k, m, present, radius)
        want = tde.without_ok(want)
        expect = [rebuilt[i] if i in lost else bad[i] for i in range(k + m)]
    else:
        data, want = tcd.checked_decode(bad, k, m, present, radius)
        want = tde.without_ok(want)
        expect = [data[i] if i < k else bad[i] for i in range(k + m)]
    assert got == want, (route_id(route), shift, n)
    for i in range(k + m):
        if call == "decode" and i in lost and i >= k:
            continue                                         # passed as NULL
        assert (after[i] == expect[i]).all(), (route_id(route), shift, n, i)
    # nothing outside the shards' columns is written
    assert torch.equal(buf[:, :shift], before[:, :shift]) and torch.equal(buf[:, shift + n:], before[:, shift + n:])
    return got


@pytest.fixture(scope="module")
def clean_sets():
    cache = {}

    def get(k, m, n):
        if (k, m, n) not in cache:
            cache[(k, m, n)] = tde.random_set(k, m, n, seed=(k * 64 + m) * 1_000_003 + n)
        return cache[(k, m, n)]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("shift", [0, 1])
@pytest.mark.parametrize("route", ROUTES, ids=route_id)
def test_device_route_every_placement_and_length(cuda, swec, clean_sets, route, shift):
    """The corpus at every shard length through one route, aligned (vector path) and off by one (byte path)."""
    torch = cuda
    call, k, m, lost, radius, _ = route
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    cases = 0
    for n in LENGTHS:
        clean = clean_sets(k, m, n)
        for j, (name, pl) in enumerate(corpus(n, k, m, radius, lost).items()):
            bad = apply(clean, pl, seed=n + j)
            bad = [None if i in lost else s for i, s in enumerate(bad)]
            assert check_route(torch, enc, route, bad, shift)["damaged_columns"] > 0, (n, name)
            cases += 1
    assert cases == 38
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("route", [r for r in ROUTES if r[0] in ("locate", "rebuild", "decode")], ids=route_id)
def test_device_range_cap(cuda, swec, clean_sets, route):
    """max_ranges 0, 1 and n_ranges - 1: the ranges are the first of the full list, and n_ranges stays exact."""
    torch = cuda
    call, k, m, lost, radius, _ = route
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    n = FILE_LEN
    clean = clean_sets(k, m, n)
    pl = sorted(set().union(*[set(p) for name, p in corpus(n, k, m, radius, lost).items()
                              if name in ("runs", "interleave", "seams")]))
    pl = [(c, ids) for c, ids in pl if not any(c == c2 and ids != i2 for c2, i2 in pl)]
    bad = [None if i in lost else s for i, s in enumerate(apply(clean, pl, seed=5))]
    full, _, _ = run_route(torch, enc, route, bad, 0)
    assert full["n_ranges"] > 8
    for cap in (0, 1, full["n_ranges"] - 1):
        got, _, _ = run_route(torch, enc, route, bad, 0, max_ranges=cap)
        assert got == {**full, "ranges": full["ranges"][:cap]}, cap
    enc.close()


@pytest.mark.gpu
def test_device_runs_merge_across_the_piece_boundary(cuda, swec):
    """RS(10,4), shards of 256 MiB + 8 KiB: damage either side of the piece boundary and one shard's run across it.
    The set is zero outside a codeword window around the boundary, so the oracle runs on the window alone."""
    torch = cuda
    if tde.free_bytes(torch) < 6 << 30:
        pytest.skip("needs 6 GiB of free device memory")
    k, m = 10, 4
    n = PIECE + 2 * PAGE
    lo = PIECE - 6 * PAGE
    win = tde.random_set(k, m, n - lo, seed=77)
    pl = ([(PIECE - 1, (0,)), (PIECE, (0,)), (PIECE - 17, (12,)), (PIECE + 16, (12,)), (PIECE - 3, (1, 2)),
           (PIECE + 5, (1, 2)), (n - 1, (13,)), (lo, (4,))]
          + [(p * PAGE + 99, (7,)) for p in range(PIECE // PAGE - 4, PIECE // PAGE + 2)])
    bad_win = apply(win, [(c - lo, ids) for c, ids in pl], seed=9)
    cols, a, b, _, _, _ = do.decode_columns(bad_win, k, m, 1)
    want = tde.without_ok(do.report(n, k + m, cols + lo, a, b))
    assert want["shards"][0][1:] == (PIECE - 1, PIECE) and any(o < PIECE < o + ln for s, o, ln in want["ranges"])
    buf = torch.zeros((k + m, n), dtype=torch.uint8, device="cuda")
    for i in range(k + m):
        buf[i, lo:] = torch.from_numpy(bad_win[i]).cuda()
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    got = enc.locate_damage_device([buf[i].data_ptr() for i in range(k + m)], n, radius=1)
    assert got == want
    got = enc.correct_damage_device([buf[i].data_ptr() for i in range(k + m)], n, radius=1)
    assert got == want
    fixed = locate_expected(bad_win, k, m, 1)[1]
    assert all((buf[i, lo:].cpu().numpy() == fixed[i]).all() for i in range(k + m))
    assert int(buf[:, :lo].count_nonzero()) == 0
    enc.close()
    del buf
    torch.cuda.empty_cache()


def _names_child():
    """Runs in a fresh process: one call per route of 4,099 columns with one wrong byte in the route's first role
    shard, under torch.profiler.  Prints RESULT <json>: per route, the sorted (MT, MODE) that ran."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    import seaweedfs_b200.erasure_coding as ec
    out = {}
    n = 4099
    for route in ROUTES:
        call, k, m, lost, radius, _ = route
        bad = tde.random_set(k, m, n, seed=k + m)
        bad[roles(k, m, lost)["A"]][1000] ^= 0x40
        bad = [None if i in lost else s for i, s in enumerate(bad)]
        enc = ec.Encoder(k, m, device=0)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            rep, _, _ = run_route(torch, enc, route, bad, 0)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
        out[route_id(route)] = {"ids": sorted({tdx.locate_id(x) for x in names} - {None}) if names else None,
                                "damaged": rep["damaged_columns"]}
        enc.close()
    print("RESULT " + json.dumps(out))


@pytest.mark.gpu
def test_each_route_runs_its_instantiation(cuda, swec):
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {here!r}]; "
            "import test_damage_runs_exhaustive as t; t._names_child()")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(next(ln for ln in r.stdout.splitlines() if ln.startswith("RESULT "))[7:])
    for route in ROUTES:
        res = got[route_id(route)]
        if res["ids"] is None:
            tkv.no_names(route_id(route))
        else:
            assert [tuple(i) for i in res["ids"]] == [route[-1]], (route_id(route), res)
        assert res["damaged"] == 1, route_id(route)


# ---------------------------------------------------------------------------------------------- GPU: file level


def pass2_stats(capfd, what):
    lines = [json.loads(x) for x in capfd.readouterr().err.splitlines() if x.startswith('{"pipe": "%s"' % what)]
    return lines


def set_direct(swec, value):
    swec._native.check(swec.lib().swec_set_option(b"file_direct_io", value))


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", FILE_CHUNKS)
@pytest.mark.parametrize("k,m", [(10, 4), (6, 3)])
def test_file_locate_and_repair_every_placement(cuda, swec, tmp_path, monkeypatch, capfd, k, m, chunk):
    """Pass 1 and pass 2 at item sizes that cut pages and warp windows: the file report equals the device call's on
    the same bytes and the oracle's; the repair leaves every file as the correction oracle does, writes no unblamed
    file, runs the pass-2 items of the restatement, and a second repair finds only what was uncorrectable."""
    torch = cuda
    ec = swec.erasure_coding
    monkeypatch.setenv("SWEC_FILE_CHUNK", str(chunk))
    monkeypatch.setenv("SWEC_PIPE_STATS", "1")
    ctx = ec.ECContext(k, m)
    enc = ec.Encoder(k, m, device=0)
    clean = tde.random_set(k, m, FILE_LEN, seed=k * 31 + chunk)
    base = str(tmp_path / "9")
    paths = tdr.shard_paths(base, k + m)
    for j, (name, pl) in enumerate(corpus(FILE_LEN, k, m, 1).items()):
        bad = apply(clean, pl, seed=chunk + j)
        want, fixed = locate_expected(bad, k, m, 1)
        tdr.write_set(base, bad)
        tdr.age(paths)
        dev, _, _ = run_route(torch, enc, ("locate", k, m, (), 1, None), bad, 0)
        assert dev == want, name
        loc = ec.locate_ec_damage(base, ctx=ctx)
        assert loc == {"ok": False, **want}, name
        capfd.readouterr()
        rep = ec.repair_ec_damage(base, ctx=ctx)
        assert rep == {"ok": want["uncorrectable_columns"] == 0, **want}, name
        stats = pass2_stats(capfd, "repair_ec_damage")
        assert [(s["items"], s["chunk"]) for s in stats] == [(len(pass2_items(want["ranges"], chunk)), chunk)], name
        assert tdr.same(tdr.file_shards(base, k + m), fixed), name
        for i, p in enumerate(paths):
            if i not in want["shards"]:
                assert os.stat(p).st_mtime_ns == PAST_NS, (name, i)
        tdr.age(paths)
        again = ec.repair_ec_damage(base, ctx=ctx)
        assert again["damaged_columns"] == again["uncorrectable_columns"] == want["uncorrectable_columns"], name
        assert again["shards"] == {} and all(os.stat(p).st_mtime_ns == PAST_NS for p in paths), name
    enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("direct", [0, 3])
def test_file_repair_with_o_direct_at_item_size_768(cuda, swec, tmp_path, monkeypatch, direct):
    ec = swec.erasure_coding
    monkeypatch.setenv("SWEC_FILE_CHUNK", "768")
    k, m = 10, 4
    clean = tde.random_set(k, m, FILE_LEN, seed=3)
    pl = sorted(corpus(FILE_LEN, k, m, 1)["straddle"] + corpus(FILE_LEN, k, m, 1)["interleave"]
                + corpus(FILE_LEN, k, m, 1)["unc in runs"])
    bad = apply(clean, pl, seed=direct)
    want, fixed = locate_expected(bad, k, m, 1)
    base = str(tmp_path / "4")
    tdr.write_set(base, bad)
    old = int(os.environ.get("SWEC_FILE_DIRECT", "0") or 0) & 3
    set_direct(swec, direct)
    try:
        rep = ec.repair_ec_damage(base, ctx=ec.ECContext(k, m))
    finally:
        set_direct(swec, old)
    assert rep == {"ok": False, **want}
    assert tdr.same(tdr.file_shards(base, k + m), fixed)


# ---------------------------------------------------------------------------------------------- GPU: needles


def seam_image(rng, dat_size):
    """A volume image whose records all start and end on 256-byte seams (so on every page and item seam of the first
    data shard's block): a superblock, a gap to 256, then records of 256 .. 4352 bytes, every fifth deleted."""
    sizes = [256, 512, 768, 3840, 4096, 4352]
    dat = bytearray([3] + [0] * 255)
    live, nid = [], 1
    while True:
        total = sizes[int(rng.integers(0, len(sizes)))]
        rec = no.write_record(nid, rng.integers(0, 256, total - 41, dtype=np.uint8).tobytes(), append_at_ns=nid)
        assert len(rec) == total
        if len(dat) + len(rec) > dat_size:
            break
        if nid % 5:
            live.append((nid, len(dat), int.from_bytes(rec[12:16], "big")))
        dat += rec
        nid += 1
    dat += bytes(dat_size - len(dat))
    return np.frombuffer(bytes(dat), dtype=np.uint8).copy(), live


def needle_placement(live, walk, k, dat_size):
    """Damage at the seams of records: the first and last byte of every third record and the byte before it, wrong in
    one shard; two data shards wrong in one column of a record (uncorrectable at radius 1); one lane's mix of sets."""
    cols = {}
    for j, (_, off, size) in enumerate(live):
        if j % 3:
            continue
        end = off + no.actual_size(size, 3)
        for d in (off - 1, off, end - 1):
            i, x = walk.shard_pos(d)
            cols.setdefault(x, set()).add(i)
    _, off, _ = live[len(live) // 2]
    i, x = walk.shard_pos(off + 40)
    cols[x] = {i, (i + 1) % k}
    i, x = walk.shard_pos(live[len(live) // 3][1] + 32)
    for c in range(16):
        cols.setdefault(x // 16 * 16 + c, set()).add([0, 1, 2, 12][c % 4])
    return sorted((c, tuple(sorted(s))) for c, s in cols.items())


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [256, 768, 4352])
def test_handle_needles_on_record_seams(cuda, swec, tmp_path, monkeypatch, capfd, chunk):
    """locate_needle_damage and repair_needle_damage through the handle: every needle's mask and counts and the
    unowned counts are the oracle's, the files end up as the correction oracle leaves them, the pass-2 items are the
    restatement's, and every needle without uncorrectable bytes checks ok afterwards."""
    ec = swec.erasure_coding
    monkeypatch.setenv("SWEC_FILE_CHUNK", str(chunk))
    monkeypatch.setenv("SWEC_PIPE_STATS", "1")
    k, m = 10, 4
    dat, live = seam_image(np.random.default_rng(chunk), 2_600_000)
    base, dat, live = tnd.generated_volume(swec, tmp_path, "6", dat=dat, live=live)
    walk = tnd.Striping(k, len(dat), tnd.GIB, tnd.MIB)
    shards = apply(tdr.file_shards(base, k + m), needle_placement(live, walk, k, len(dat)), seed=chunk)
    tdr.write_set(base, shards)
    vol = ec.EcVolume(base)
    info = vol.info()
    want = tnd.handle_expected(base, k, m, 1, live, info["shard_dat_size"])
    rep, per, unowned = want
    assert rep["uncorrectable_columns"] > 0 and rep["damaged_columns"] > len(live) // 2
    fixed = tdr.correct(shards, k, m, 1)
    for call in (vol.locate_needle_damage, vol.repair_needle_damage):
        capfd.readouterr()
        res = call()
        ok = res.pop("ok")
        tnd.handle_compare({**res, "ok": False}, ({**rep, "ok": False}, per, unowned), live)
        items = [(s["items"], s["chunk"]) for s in pass2_stats(capfd, call.__name__)]
        assert items == [(len(pass2_items(rep["ranges"], chunk)), chunk)], call.__name__
        if call == vol.locate_needle_damage:
            assert tdr.same(tdr.file_shards(base, k + m), shards)
    assert not ok
    assert tdr.same(tdr.file_shards(base, k + m), fixed)
    for r in res["needles"]:
        if not r["uncorrectable_bytes"]:
            assert r["status"] == 0, r
    lost = {r["needle_id"] for r in res["needles"] if r["uncorrectable_bytes"]}
    _, _, errors = vol.scrub_needles(6)
    bad = {int(e.split()[1]) for e in errors if e.startswith("needle ")}
    assert bad <= lost
    vol.close()
