"""The file-level pipeline (seaweedfs_b200/csrc/ec_files.cc) at every seam of the stripe geometry, the staging ring and the
I/O cuts: ec.encode (swec_generate_ec_files), ec.rebuild (swec_rebuild_ec_files[_checked]), the parity scrub
(swec_verify_ec_files), locate and in-place repair (swec_locate_ec_damage, swec_repair_ec_damage) and ec.decode
(swec_write_dat_file_checked, and the plain copy swec_write_dat_file).

A volume is cut into items: rows of large blocks at the slot pitch, small rows several to a slot (row by row when a small
block is larger than a slot), the tail row last; the column walks of verify, locate, repair and rebuild cut the shards at
the slot pitch.  item_plan() restates the cut in Python; the sizes below are picked from it so that they land on the
seams, and the item count of every generate is checked against it (SWEC_PIPE_STATS).  Every expected value comes from an
existing oracle: shard bytes from oracle.encode_dat_image, .dat bytes from oracle.write_dat_image, locate / repair reports
and corrected bytes from damage_oracle.locate and test_damage_repair.correct, checked decode and checked rebuild reports
from test_checked_decode.checked_decode, verify counts from the distinct 16-byte vectors of damage_oracle.syndromes.

cpu: the item plan on hand-computed cases; the plain .dat copy over the whole size x block grid and across its 8 MiB
piece cut.
gpu: generate + clean verify over slot pitches 4096, 4352 (17 x 256: every stream after the first is misaligned for
O_DIRECT) and 65536 x five block pairs x every seam size, RS(10,4) in full and RS(6,3), RS(20,12), RS(1,3), RS(31,1) on a
reduced grid; on RS(10,4) and RS(6,3), one block pair per pitch, verify with damage, rebuild, checked rebuild, locate and
repair (the ring wraps) and checked decode at every size, the empty volume included; the reference's 1 MiB ragged-rebuild
quirk; stage_slots 2, 3, 5, 16; read and write pieces shorter than an item; file_direct_io 0-3 with O_DIRECT shown in
use through /proc/self/fdinfo; a parked ring full of stale bytes; the table-to-specialised-kernel switch of a rebuild
(torch.profiler, in a child process); the volume-level generate reaching the pipeline."""
import ctypes as C
import json
import math
import mmap
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import damage_oracle as do  # noqa: E402
import test_checked_decode as tcd  # noqa: E402
import test_damage_repair as tdr  # noqa: E402

ROOT = os.path.dirname(HERE)
MIB = 1 << 20
PAST_NS = tdr.PAST_NS
O_DIRECT = 0o40000                     # x86-64 open flag, as /proc/<pid>/fdinfo prints it (octal)
PITCHES = (4096, 4352, 65536)
RATIOS = ((10, 4), (6, 3), (20, 12), (1, 3), (31, 1))
DEEP_PAIR = {4096: "short", 4352: "row", 65536: "quarter"}    # the block pair of the deep checks at each pitch


# ---------------------------------------------------------------------------------------------- the item plan


def file_chunk(span, cap):
    """The slot pitch of a pipeline over streams of `span` bytes: the configured chunk, or less, in 256-byte units."""
    return max(256, (min(cap, max(span, 1)) + 255) & ~255)


def geometry(dat_size, k, large, small):
    """(large rows, full small rows, tail bytes) of encodeDatFile's striping."""
    large_rows = dat_size // (large * k)
    rem = dat_size - large_rows * large * k
    small_rows = rem // (small * k)
    return large_rows, small_rows, rem - small_rows * small * k


def shard_size(dat_size, k, large, small):
    large_rows, small_rows, tail = geometry(dat_size, k, large, small)
    return large_rows * large + small_rows * small + (small if tail else 0)


def decode_cols(dat_size, k, large, small):
    """Columns the decode reads: the tail row counts only as far as shard 0 holds it."""
    large_rows, small_rows, tail = geometry(dat_size, k, large, small)
    return large_rows * large + small_rows * small + min(tail, small)


def generate_chunk(large, small, cap):
    return file_chunk(max(large, small), cap)


def decode_chunk(dat_size, k, large, small, cap):
    return file_chunk(decode_cols(dat_size, k, large, small), cap)


def item_plan(dat_size, k, large, small, chunk, decode=False):
    """[(shard offset, length, stripe rows)] of swec_generate_ec_files (decode=False) or of the checked decode: large rows
    cut at the slot size, then small rows chunk // small to a slot (row by row when small > chunk), the tail row last.
    Generate reads the tail row as a whole small row (zero past EOF); the decode takes the columns shard 0 gives it."""
    large_rows, small_rows, tail = geometry(dat_size, k, large, small)
    items = []
    for r in range(large_rows):
        for o in range(0, large, chunk):
            items.append((r * large + o, min(chunk, large - o), (r,)))
    widths = [small] * small_rows + ([min(tail, small) if decode else small] if tail else [])
    base = large_rows * large
    if small > chunk:
        for j, w in enumerate(widths):
            for o in range(0, w, chunk):
                items.append((base + j * small + o, min(chunk, w - o), (large_rows + j,)))
        return items
    per = max(1, chunk // small)
    for first in range(0, len(widths), per):
        ws = widths[first:first + per]
        items.append((base + first * small, sum(ws), tuple(range(large_rows + first, large_rows + first + len(ws)))))
    return items


def block_pairs(c):
    """(name, large, small) relative to the slot pitch c."""
    wide = (5 * c // 2 + 255) // 256 * 256                  # about 2.5 c, 256-aligned
    return [("quarter", 3 * c, c // 4),                     # small rows fill the slot exactly
            ("short", 3 * c + 200, 1000),                   # the slot is not filled; large rows end on a short item
            ("equal", c, c),
            ("row", 2 * (c + 256), c + 256),                # row by row, with a 256-byte second item
            ("wide", 4 * wide, wide)]


def pair(c, name):
    return next(p for p in block_pairs(c) if p[0] == name)[1:]


def rows_for_items(n, k, small, chunk):
    """Small rows after which the small part of a plan has more than n items."""
    rows = 1
    while len(item_plan(rows * k * small, k, 10 ** 12, small, chunk)) <= n:
        rows += 1
    return rows


def ring_size(k, large, small, chunk, slots=3):
    """A large row plus small rows whose plan has more than 2*slots+1 items.  Small rows after the last large row are
    fewer than large / small (more would make another large row), so pairs with large close to small add large rows."""
    rows = min(rows_for_items(2 * slots + 1, k, small, chunk), (large - 1) // small)
    d = large * k + rows * k * small
    while len(item_plan(d, k, large, small, chunk)) <= 2 * slots + 1:
        d += large * k
    return d


def seam_sizes(k, large, small, chunk, slots=3):
    """Every .dat size of the geometry grid: the edges of the first small row and of the shard boundaries, a row of
    large blocks +-1, ring_size() with three tails, two large rows + 3 small rows + 5."""
    s, big = small, large * k
    out = {0, 1, s - 1, s, s + 1, k * s - 1, k * s, k * s + 1, (k - 1) * s + 1}
    out |= {j * s for j in range(1, k)}
    out |= {big - 1, big, big + 1}
    out |= {ring_size(k, large, small, chunk, slots) + t for t in (0, s, (k - 1) * s + 17)}
    out.add(2 * big + 3 * k * s + 5)
    return sorted(out)


def size_with_items(n, k, large, small, chunk):
    """The smallest .dat size (17-byte tail) whose generate plan has exactly n items."""
    for a in range(64):
        for b in range(large // small + 2):
            d = a * large * k + b * k * small + 17
            if len(item_plan(d, k, large, small, chunk)) == n:
                return d
    raise AssertionError("no size with %d items" % n)


# ---------------------------------------------------------------------------------------------- files and knobs


def read_shards(base, n):
    return [np.fromfile(base + ".ec%02d" % i, dtype=np.uint8) for i in range(n)]


def write_set(base, shards, skip=()):
    for i, s in enumerate(shards):
        if i not in skip:
            s.tofile(base + ".ec%02d" % i)


def same(a, b):
    return len(a) == len(b) and all(len(x) == len(y) and (x == y).all() for x, y in zip(a, b))


def random_dat(size, seed, fill=None):
    if fill is not None:
        return np.full(size, fill, dtype=np.uint8)
    return np.random.default_rng(seed).integers(0, 256, size, dtype=np.uint8)


def generate(ec, capfd, base, dat, k, m, large, small):
    """swec_generate_ec_files with SWEC_PIPE_STATS set (by the caller): returns its pipeline's stats line."""
    dat.tofile(base + ".dat")
    capfd.readouterr()
    ec.generate_ec_files(base, math.gcd(large, small), large, small, ec.ECContext(k, m))
    lines = [json.loads(x) for x in capfd.readouterr().err.splitlines() if x.startswith('{"pipe": "generate_ec_files"')]
    assert len(lines) == 1, lines
    return lines[0]


def expected_shards(oracle, dat, k, m, large, small):
    return oracle.encode_dat_image(dat, k=k, m=m, buffer_size=math.gcd(large, small), large=large, small=small)


def vector_counts(shards, k, m):
    """Per parity row: the distinct 16-byte vectors with a differing byte (what swec_verify_ec_files counts)."""
    s = do.syndromes(shards, k, m)
    return [len(np.unique(np.flatnonzero(s[:, p]) // 16)) for p in range(m)]


class Edits:
    """Damage of one wrong shard per column: column -> shard id (the first claim of a column wins)."""

    def __init__(self, size):
        self.size, self.cols = size, {}

    def put(self, col, sid):
        if 0 <= col < self.size and col not in self.cols:
            self.cols[int(col)] = int(sid)

    def run(self, lo, hi, sid):
        for c in range(lo, hi):
            self.put(c, sid)

    def apply(self, shards, seed):
        rng = np.random.default_rng(seed)
        out = [s.copy() for s in shards]
        for c, sid in self.cols.items():
            out[sid][c] ^= np.uint8(rng.integers(1, 256))
        return out


def set_option(swec, name, value):
    swec._native.check(swec.lib().swec_set_option(name, value))


def default_slots():
    return max(2, int(os.environ.get("SWEC_STAGE_SLOTS", "3") or 3))


def default_direct():
    return int(os.environ.get("SWEC_FILE_DIRECT", "0") or 0) & 3


@pytest.fixture
def knobs(swec, monkeypatch):
    """SWEC_PIPE_STATS on, the parked-ring cache on; stage_slots and file_direct_io back to their defaults afterwards."""
    monkeypatch.setenv("SWEC_PIPE_STATS", "1")
    monkeypatch.delenv("SWEC_NO_RING_CACHE", raising=False)
    for name in ("SWEC_FILE_IO_PIECE", "SWEC_FILE_WRITE_PIECE", "SWEC_FILE_JIT_WAIT"):
        monkeypatch.delenv(name, raising=False)
    try:
        yield monkeypatch
    finally:
        set_option(swec, b"stage_slots", default_slots())
        set_option(swec, b"file_direct_io", default_direct())


# ---------------------------------------------------------------------------------------------- O_DIRECT


def fs_type(path):
    """The filesystem type of the mount that holds path (/proc/self/mountinfo)."""
    path, best, kind = os.path.realpath(path), "", "unknown"
    with open("/proc/self/mountinfo") as f:
        for line in f:
            left, right = line.split(" - ", 1)
            point = left.split()[4]
            if (path == point or path.startswith(point.rstrip("/") + "/")) and len(point) >= len(best):
                best, kind = point, right.split()[0]
    return kind


def direct_probe(d):
    """(whether the filesystem of d takes an aligned O_DIRECT write, whether it refuses a misaligned buffer)."""
    probe = os.path.join(d, "probe")
    buf = mmap.mmap(-1, 8192)                              # page-aligned
    ok = strict = False
    try:
        fd = os.open(probe, os.O_CREAT | os.O_WRONLY | os.O_DIRECT, 0o644)
        try:
            ok = os.pwrite(fd, memoryview(buf)[:4096], 0) == 4096
            try:
                os.pwrite(fd, memoryview(buf)[256:4352], 0)
            except OSError:
                strict = True
        finally:
            os.close(fd)
    except OSError:
        pass
    finally:
        buf.close()
        if os.path.exists(probe):
            os.remove(probe)
    return ok, ok and strict


def direct_dir(tmp_path):
    """(a directory for the O_DIRECT cases, every candidate with its filesystem, whether the chosen one refuses a
    misaligned O_DIRECT buffer).  Candidates: tmp_path, then a directory under the repository's .pytest_cache/.  One
    that refuses misaligned buffers (ext4, xfs) wins over one that only accepts O_DIRECT (9p, tmpfs); None when no
    candidate accepts O_DIRECT."""
    found, tried = [], []
    for d in (str(tmp_path), os.path.join(ROOT, ".pytest_cache")):
        try:
            os.makedirs(d, exist_ok=True)
            d = tempfile.mkdtemp(prefix="odirect-", dir=d) if d != str(tmp_path) else d
        except OSError:
            continue
        ok, strict = direct_probe(d)
        tried.append("%s (%s%s)" % (d, fs_type(d), ", strict" if strict else ", O_DIRECT" if ok else ""))
        if ok:
            found.append((strict, d))
        elif d != str(tmp_path):
            shutil.rmtree(d, ignore_errors=True)
    if not found:
        return None, tried, False
    strict, best = next((f for f in found if f[0]), found[0])
    for _, d in found:
        if d != best and d != str(tmp_path):
            shutil.rmtree(d, ignore_errors=True)
    return best, tried, strict


class DirectWatch:
    """While a call runs, polls /proc/self/fd and /proc/self/fdinfo for descriptors on paths under `prefix`: the
    (access mode, O_DIRECT) pairs seen.  ctypes releases the GIL during the call, so the poller runs alongside it."""

    def __init__(self, prefix):
        self.prefix = os.path.realpath(prefix)
        self.seen = set()
        self._stop = threading.Event()

    def _poll(self):
        while not self._stop.is_set():
            for fd in os.listdir("/proc/self/fd"):
                try:
                    path = os.readlink("/proc/self/fd/" + fd)
                    if not path.startswith(self.prefix):
                        continue
                    with open("/proc/self/fdinfo/" + fd) as f:
                        flags = next(int(x.split()[1], 8) for x in f if x.startswith("flags:"))
                except (OSError, StopIteration):
                    continue
                self.seen.add((flags & 3, bool(flags & O_DIRECT)))
            time.sleep(0.0005)

    def __enter__(self):
        self._t = threading.Thread(target=self._poll, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()
        return False


# ---------------------------------------------------------------------------------------------- CPU


def test_item_plan_hand_computed():
    # k = 2, large 128, small 16, slot 64: one large row in two items, then four small rows that fill one slot exactly
    assert item_plan(256 + 4 * 32, 2, 128, 16, 64) == [(0, 64, (0,)), (64, 64, (0,)), (128, 64, (1, 2, 3, 4))]
    assert item_plan(256 + 5 * 32, 2, 128, 16, 64)[2:] == [(128, 64, (1, 2, 3, 4)), (192, 16, (5,))]
    # small 300 > slot 256: the large row in three items, each small row in two, the tail row as a whole row
    d = 2 * 600 + 2 * 300 + 10
    assert item_plan(d, 2, 600, 300, 256) == [(0, 256, (0,)), (256, 256, (0,)), (512, 88, (0,)),
                                              (600, 256, (1,)), (856, 44, (1,)), (900, 256, (2,)), (1156, 44, (2,))]
    assert item_plan(d, 2, 600, 300, 256, decode=True)[-1] == (900, 10, (2,))
    assert decode_cols(d, 2, 600, 300) == 910 and shard_size(d, 2, 600, 300) == 1200
    # a tail alone: one item of a whole small row, of 5 columns for the decode
    assert item_plan(5, 3, 100, 10, 256) == [(0, 10, (0,))]
    assert item_plan(5, 3, 100, 10, 256, decode=True) == [(0, 5, (0,))]
    assert item_plan(0, 3, 100, 10, 256) == []
    # the tail ends exactly on a shard boundary: shard 0 holds a whole block of it
    assert item_plan(30 + 10, 3, 100, 10, 256, decode=True) == item_plan(30 + 10, 3, 100, 10, 256) == [(0, 20, (0, 1))]
    assert file_chunk(0, 4096) == 256 and file_chunk(4097, 1 << 20) == 4352 and file_chunk(1 << 30, 4352) == 4352
    # the ring-wrap sizes of the grid: more than 2*slots+1 items, small rows included where the pair allows them
    for c in PITCHES:
        for name, large, small in block_pairs(c):
            d = ring_size(10, large, small, c)
            plan = item_plan(d, 10, large, small, c)
            assert len(plan) > 7 and d in seam_sizes(10, large, small, c), name


def _plain_copy_case(ec, oracle, tmp, k, large, small, dat_size, seed):
    dat = random_dat(dat_size, seed)
    shards = expected_shards(oracle, dat, k, 1, large, small)[:k]
    base = os.path.join(tmp, "p")
    write_set(base, shards)
    ec.write_dat_file(os.path.join(tmp, "out"), dat_size, [base + ".ec%02d" % i for i in range(k)], data_shards=k,
                      large_block=large, small_block=small)
    got = np.fromfile(os.path.join(tmp, "out.dat"), dtype=np.uint8)
    want = oracle.write_dat_image(shards, dat_size, k=k, large=large, small=small)
    assert len(got) == dat_size and (got == want).all() and (want == dat).all(), (k, large, small, dat_size)


@pytest.mark.parametrize("c", PITCHES)
def test_plain_copy_over_the_grid(swec, oracle, tmp_path, c):
    """swec_write_dat_file (no GPU) over every block pair and seam size of the geometry grid."""
    ec = swec.erasure_coding
    for name, large, small in block_pairs(c):
        for d in seam_sizes(10, large, small, c):
            _plain_copy_case(ec, oracle, str(tmp_path), 10, large, small, d, seed=d + c)


def test_plain_copy_across_the_8_mib_piece(swec, oracle, tmp_path):
    ec = swec.erasure_coding
    large = (8 << 20) + 3 * 4096 + 256                   # a block longer than the copy's 8 MiB piece
    _plain_copy_case(ec, oracle, str(tmp_path), 2, large, 4096, 2 * large + 3 * 2 * 4096 + 5, seed=88)


# ---------------------------------------------------------------------------------------------- GPU: the geometry grid


def _grid_point(ec, oracle, capfd, base, k, m, c, large, small, d):
    dat = random_dat(d, seed=d * 31 + k * 7 + c)
    stats = generate(ec, capfd, base, dat, k, m, large, small)
    plan = item_plan(d, k, large, small, generate_chunk(large, small, c))
    assert (stats["items"], stats["chunk"]) == (len(plan), generate_chunk(large, small, c)), (k, m, c, large, small, d)
    clean = read_shards(base, k + m)
    assert len(clean[0]) == ec.expected_shard_size(d, k, large, small) == shard_size(d, k, large, small)
    assert same(clean, expected_shards(oracle, dat, k, m, large, small)), (k, m, c, large, small, d)
    assert ec.verify_ec_files(base, ctx=ec.ECContext(k, m)) == (True, [0] * m), (k, m, c, large, small, d)
    return dat, clean


GRID = [(10, 4, c, name) for c in PITCHES for name, *_ in block_pairs(c)] + \
       [(k, m, 4096, name) for k, m in RATIOS[1:] for name in ("quarter", "short", "row")]


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,c,name", GRID)
def test_generate_and_verify_grid(cuda, swec, oracle, tmp_path, capfd, knobs, k, m, c, name):
    """Generate: every shard byte for byte, the item count of the plan; a clean verify."""
    ec = swec.erasure_coding
    knobs.setenv("SWEC_FILE_CHUNK", str(c))
    large, small = pair(c, name)
    for d in seam_sizes(k, large, small, c):
        _grid_point(ec, oracle, capfd, str(tmp_path / "g"), k, m, c, large, small, d)


def _check_verify_damage(ec, base, clean, k, m, c):
    size, n = len(clean[0]), k + m
    chunk = file_chunk(size, c)
    e = Edits(size)
    for j, o in enumerate(range(0, size, chunk)):         # the first and last byte of every item
        e.put(o, j % n)
        e.put(min(o + chunk, size) - 1, (j + 1) % n)
    if size % 16:                                         # inside the tail's partial 16-byte vector
        e.put(size - size % 16 + (size % 16) // 2, n - 1)
    parity_only = Edits(size)
    parity_only.put(size // 2, k + m // 2)
    for edits in (e, parity_only):
        damaged = edits.apply(clean, seed=size + len(edits.cols))
        write_set(base, damaged)
        counts = vector_counts(damaged, k, m)
        assert ec.verify_ec_files(base, ctx=ec.ECContext(k, m)) == (not any(counts), counts), (k, m, c, size)
    write_set(base, clean)


def _check_rebuild(ec, base, clean, k, m):
    """One data shard, one parity shard and m mixed ones lost.  Shards of the grid stay at or under 1 MiB, below the
    ragged-length quirk, which test_ragged_rebuild_quirk covers."""
    size = len(clean[0])
    assert size <= MIB
    for lost in ((min(3, k - 1),), (k,), tuple(range(m // 2)) + tuple(range(k, k + m - m // 2))):
        for i in lost:
            os.remove(base + ".ec%02d" % i)
        assert ec.rebuild_ec_files(base, ctx=ec.ECContext(k, m)) == sorted(lost)
        assert same(read_shards(base, k + m), clean), (k, m, size, lost)


def _check_checked_rebuild(ec, base, clean, k, m, c):
    size, n = len(clean[0]), k + m
    lost = (1 % k,)
    present = tcd.mask(n, lost)
    ids = [i for i in range(n) if present[i]]
    chunk = file_chunk(size, c)
    e = Edits(size)
    for j, o in enumerate(range(chunk, size, chunk)):     # both sides of every item seam
        e.put(o - 1, ids[j % len(ids)])
        e.put(o, ids[(j + 5) % len(ids)])
    e.put(size - 1, ids[-1])
    damaged = e.apply(clean, seed=size + 3)
    write_set(base, damaged)
    os.remove(base + ".ec%02d" % lost[0])
    rep = ec.rebuild_ec_files_checked(base, ctx=ec.ECContext(k, m))
    _, want = tcd.checked_decode([d if present[i] else None for i, d in enumerate(damaged)], k, m, present)
    assert rep == {"rebuilt": list(lost), **want}, (k, m, c, size)
    assert (np.fromfile(base + ".ec%02d" % lost[0], dtype=np.uint8) == clean[lost[0]]).all()
    write_set(base, clean)


def _check_locate_repair(ec, base, clean, k, m, c):
    size, n = len(clean[0]), k + m
    chunk = file_chunk(size, c)
    e = Edits(size)
    seams = list(range(chunk, size, chunk))
    for j, o in enumerate(seams[:3]):                     # runs that cross item boundaries
        e.run(o - 40, o + 40, (j + 3) % n)
    e.run(size - 30, size, n - 2)                         # the clipped last page
    for j, o in enumerate(range(0, size, chunk)):         # a byte in every item: 2*slots+1 and more when there are
        e.put(o + chunk // 2, j % n)
    damaged = e.apply(clean, seed=size + 5)
    write_set(base, damaged)
    paths = tdr.shard_paths(base, n)
    tdr.age(paths)
    want = do.locate(damaged, k, m)
    assert ec.locate_ec_damage(base, ctx=ec.ECContext(k, m)) == {**want, "ok": want["damaged_columns"] == 0}
    assert tdr.mtimes(paths) == [PAST_NS] * n
    rep = ec.repair_ec_damage(base, ctx=ec.ECContext(k, m))
    assert rep == {**want, "ok": want["uncorrectable_columns"] == 0}, (k, m, c, size)
    fixed = read_shards(base, n)
    assert same(fixed, tdr.correct(damaged, k, m)) and same(fixed, clean), (k, m, c, size)
    assert [t != PAST_NS for t in tdr.mtimes(paths)] == [i in want["shards"] for i in range(n)]


def _check_checked_decode(ec, base, dat, clean, k, m, c, large, small):
    d, n = len(dat), k + m
    cols = decode_cols(d, k, large, small)
    plan = item_plan(d, k, large, small, decode_chunk(d, k, large, small, c), decode=True)
    e = Edits(cols)
    for j, (off, ln, _) in enumerate(plan):               # one wrong data byte at both ends of every item
        e.put(off, j % k)
        e.put(off + ln - 1, (j + 1) % k)
    damaged = e.apply(clean, seed=d + 9)
    out = base + "-out"
    # data shards go first: with m = 4, 0 and 1 (k + 2 present, radius 1), then 0 .. 2 (k + 1: detection only), then
    # 0 .. 3 (exactly k: nothing to check against)
    cases = [((), damaged), (tuple(range(m - 2)), damaged), (tuple(range(m - 1)), clean),
             (tuple(range(m - 1)), damaged), (tuple(range(m)), clean)]
    for lost, shards in cases:
        present = tcd.mask(n, lost)
        write_set(base, shards)
        if os.path.exists(out + ".dat"):
            os.remove(out + ".dat")
        names = [base + ".ec%02d" % i if present[i] else None for i in range(n)]
        _, want = tcd.checked_decode([s[:cols] if present[i] else None for i, s in enumerate(shards)], k, m, present)
        if want["uncorrectable_columns"]:                 # k + 1 with damage in a data shard: no .dat
            with pytest.raises(Exception) as err:
                ec.write_dat_file_checked(out, d, names, data_shards=k, parity_shards=m, large_block=large,
                                          small_block=small)
            assert getattr(err.value, "name", None) == "SWEC_ERR_UNCORRECTABLE", err.value
            assert {"ok": False, **err.value.report} == want and not os.path.exists(out + ".dat"), (k, m, c, d, lost)
            continue
        res = ec.write_dat_file_checked(out, d, names, data_shards=k, parity_shards=m, large_block=large,
                                        small_block=small)
        assert res == {"dat_file_size": d, **want}, (k, m, c, d, lost)
        got = np.fromfile(out + ".dat", dtype=np.uint8)
        assert len(got) == d and (got == dat).all(), (k, m, c, d, lost)
    write_set(base, clean)


DEEP = [(k, m, c) for k, m in RATIOS[:2] for c in PITCHES]


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,c", DEEP)
def test_every_call_at_every_seam(cuda, swec, oracle, tmp_path, capfd, knobs, k, m, c):
    """One block pair per pitch, every seam size, the empty volume first: verify with damage, rebuild, checked rebuild,
    locate and repair, checked decode."""
    ec = swec.erasure_coding
    knobs.setenv("SWEC_FILE_CHUNK", str(c))
    large, small = pair(c, DEEP_PAIR[c])
    base = str(tmp_path / "v")
    for d in seam_sizes(k, large, small, c):
        dat, clean = _grid_point(ec, oracle, capfd, base, k, m, c, large, small, d)
        _check_verify_damage(ec, base, clean, k, m, c)
        _check_rebuild(ec, base, clean, k, m)
        _check_checked_rebuild(ec, base, clean, k, m, c)
        _check_locate_repair(ec, base, clean, k, m, c)
        _check_checked_decode(ec, base, dat, clean, k, m, c, large, small)


@pytest.mark.gpu
def test_ragged_rebuild_quirk(cuda, swec, tmp_path):
    """The reference reads 1 MiB buffers: a 2 MiB shard rebuilds, a 2 MiB + 1 one fails and leaves no output file."""
    ec = swec.erasure_coding
    for length, ok in ((2 * MIB, True), (2 * MIB + 1, False)):
        clean = tdr.random_set(10, 4, length, seed=length)
        base = str(tmp_path / ("q%d" % length))
        write_set(base, clean, skip=(2,))
        if ok:
            assert ec.rebuild_ec_files(base) == [2]
            assert same(read_shards(base, 14), clean)
        else:
            with pytest.raises(swec.SwecError) as e:
                ec.rebuild_ec_files(base)
            assert e.value.name == "SWEC_ERR_SHARD_SIZE" and not os.path.exists(base + ".ec02")


# ---------------------------------------------------------------------------------------------- GPU: knob sweeps


SWEEP_C = 4096
SWEEP_PAIR = pair(SWEEP_C, "short")


def _pipeline_round(ec, oracle, capfd, base, d, k=10, m=4, c=SWEEP_C, blocks=SWEEP_PAIR, rebuild=False):
    """generate (bytes and items), clean verify, repair of a byte in every column-walk item, checked decode with a wrong
    data byte at every decode seam; with `rebuild`, a rebuild of two lost shards."""
    large, small = blocks
    dat, clean = _grid_point(ec, oracle, capfd, base, k, m, c, large, small, d)
    size, n = len(clean[0]), k + m
    chunk = file_chunk(size, c)
    e = Edits(size)
    for j, o in enumerate(range(0, size, chunk)):
        e.put(o + (j * 37) % min(chunk, size - o), j % n)
    damaged = e.apply(clean, seed=d)
    write_set(base, damaged)
    want = do.locate(damaged, k, m)
    assert ec.repair_ec_damage(base, ctx=ec.ECContext(k, m)) == {**want, "ok": True}
    assert same(read_shards(base, n), clean), d
    _check_checked_decode(ec, base, dat, clean, k, m, c, large, small)
    if rebuild:
        _check_rebuild(ec, base, clean, k, m)


@pytest.mark.gpu
@pytest.mark.parametrize("slots", [2, 3, 5, 16])
def test_stage_slots(cuda, swec, oracle, tmp_path, capfd, knobs, slots):
    """Plans of 1, slots-1, slots, slots+1 and 3*slots+1 items on rings of 2 to 16 slots."""
    ec = swec.erasure_coding
    knobs.setenv("SWEC_FILE_CHUNK", str(SWEEP_C))
    set_option(swec, b"stage_slots", slots)
    large, small = SWEEP_PAIR
    chunk = generate_chunk(large, small, SWEEP_C)
    for n in sorted({1, slots - 1, slots, slots + 1, 3 * slots + 1}):
        d = size_with_items(n, 10, large, small, chunk)
        _pipeline_round(ec, oracle, capfd, str(tmp_path / "s"), d)


@pytest.mark.gpu
@pytest.mark.parametrize("read_piece", [4096, 12288])
@pytest.mark.parametrize("write_piece", [4096, 12288])
def test_read_and_write_pieces(cuda, swec, oracle, tmp_path, capfd, knobs, read_piece, write_piece):
    """At a 64 KiB slot, reads and writes are cut into pieces and the last piece of an item is short."""
    ec = swec.erasure_coding
    c = 65536
    knobs.setenv("SWEC_FILE_CHUNK", str(c))
    knobs.setenv("SWEC_FILE_IO_PIECE", str(read_piece))
    knobs.setenv("SWEC_FILE_WRITE_PIECE", str(write_piece))
    large, small = pair(c, "short")
    d = 2 * large * 10 + 70 * small * 10 + 5
    _pipeline_round(ec, oracle, capfd, str(tmp_path / "p"), d, c=c, blocks=(large, small), rebuild=True)


DIRECT_ALIGNED = (3 * 4096, 4096)      # a block pair whose tail-row reads start 4 KiB-aligned


def direct_reads_across_eof(d, k, large, small, chunk, piece):
    """The read pieces of generate's tail row that the O_DIRECT descriptor takes (.dat offset, length and slot buffer
    all 4 KiB-aligned; the slot buffer of stream i starts at i * chunk) and that reach past EOF: (offset, length).
    Their short O_DIRECT read at EOF goes on on the buffered descriptor, and the rest is zero-filled."""
    large_rows, small_rows, tail = geometry(d, k, large, small)
    if not tail:
        return []
    row = large_rows * large * k + small_rows * small * k           # .dat offset of the tail row
    if small > chunk:                                               # row by row: stream i holds block i from 0
        reads = [(row + small * i + o, min(chunk, small - o), i * chunk) for i in range(k) for o in range(0, small, chunk)]
    else:                                                           # the tail row is row j of its item
        j = len(item_plan(d, k, large, small, chunk)[-1][2]) - 1
        reads = [(row + small * i, small, i * chunk + j * small) for i in range(k)]
    out = []
    for off, ln, dst in reads:
        for o in range(0, ln, piece):
            n = min(piece, ln - o)
            if (off + o) % 4096 == 0 and n % 4096 == 0 and (dst + o) % 4096 == 0 and off + o + n > d:
                out.append((off + o, n))
    return out


def test_direct_sizes_read_across_eof():
    """The .dat sizes of test_file_direct_io that are not whole 4 KiB pages send an aligned O_DIRECT read past EOF at
    both pitches and both read pieces."""
    large, small = DIRECT_ALIGNED
    for c in (4096, 4352):
        for piece in (2 << 20, 4096):
            sizes = direct_sizes(large, small)
            assert any(d % 4096 for d in sizes) and any(d % 4096 == 0 for d in sizes)
            assert all(not direct_reads_across_eof(d, 10, large, small, c, piece) for d in sizes if d % 4096 == 0)
            assert any(direct_reads_across_eof(d, 10, large, small, c, piece) for d in sizes if d % 4096), (c, piece)
    # stream 0 alone is aligned at pitch 4352: a tail shorter than one block straddles there, a longer one does not
    d0 = 10 * large + 5 * 10 * small
    assert direct_reads_across_eof(d0 + 123, 10, large, small, 4352, 4096) == [(d0, 4096)]
    assert direct_reads_across_eof(d0 + 2 * 4096 + 123, 10, large, small, 4352, 4096) == []
    # at pitch 4096 every stream is aligned: block 2 straddles EOF (a short O_DIRECT read, then the buffered one), blocks
    # 3 .. 9 start past it
    d = d0 + 2 * 4096 + 123
    assert direct_reads_across_eof(d, 10, large, small, 4096, 4096) == [(d0 + i * 4096, 4096) for i in range(2, 10)]
    for c in (4096, 4352):
        for d in direct_sizes(large, small):
            straddles = any(off < d for off, _ in direct_reads_across_eof(d, 10, large, small, c, 4096))
            assert straddles == bool(d % 4096 and (c == 4096 or d - d0 < 4096)), (c, d)


def direct_sizes(large, small):
    """On 4 KiB, and with a tail ending partway into an aligned tail-row block (block 0, block 2)."""
    d0 = 10 * large + 5 * 10 * small
    return [d0, d0 + 123, d0 + 2 * 4096 + 123]


@pytest.fixture(scope="module")
def odirect(tmp_path_factory):
    d, tried, strict = direct_dir(tmp_path_factory.mktemp("odirect"))
    yield d, tried, strict
    if d and d.startswith(os.path.join(ROOT, ".pytest_cache")):
        shutil.rmtree(d, ignore_errors=True)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_file_direct_io(cuda, swec, oracle, capfd, knobs, odirect, mode):
    """file_direct_io 0-3 x slot 4096 / 4352 x read piece default / 4096, .dat sizes on and off 4 KiB: the bytes of the
    oracle, and O_DIRECT descriptors really in use.  The 'quarter' pair reads the .dat at offsets off 4 KiB; the
    aligned pair DIRECT_ALIGNED sends aligned O_DIRECT reads past EOF (direct_reads_across_eof), so the fallback to the
    buffered descriptor and the zero fill run.  Where the filesystem refuses a misaligned O_DIRECT buffer (ext4, xfs),
    a slot buffer taken to the O_DIRECT descriptor at pitch 4352 fails the call with EINVAL; where it does not (9p, for
    one), only the bytes and the descriptors are checked."""
    where, tried, strict = odirect
    if where is None:
        pytest.skip("no filesystem here accepts O_DIRECT: " + ", ".join(tried))
    if not strict:
        warnings.warn("%s (%s) takes misaligned O_DIRECT buffers: buffer alignment of the O_DIRECT path not checked"
                      % (where, fs_type(where)))
    ec = swec.erasure_coding
    set_option(swec, b"file_direct_io", mode)
    root = tempfile.mkdtemp(prefix="mode%d-" % mode, dir=where)
    seen, across_eof = set(), 0
    try:
        for c in (4096, 4352):
            knobs.setenv("SWEC_FILE_CHUNK", str(c))
            large, small = pair(c, "quarter")
            cases = [((large, small), d) for d in (large * 10 + 40 * small * 10, large * 10 + 40 * small * 10 + 4096 * 3 + 123)]
            cases += [(DIRECT_ALIGNED, d) for d in direct_sizes(*DIRECT_ALIGNED)]
            for piece in (None, 4096):
                if piece:
                    knobs.setenv("SWEC_FILE_IO_PIECE", str(piece))
                else:
                    knobs.delenv("SWEC_FILE_IO_PIECE", raising=False)
                for blocks, d in cases:
                    across_eof += len(direct_reads_across_eof(d, 10, *blocks, c, piece or (2 << 20)))
                    base = os.path.join(root, "%d-%s-%d-%d" % (c, piece, blocks[1], d))
                    with DirectWatch(root) as w:
                        _pipeline_round(ec, oracle, capfd, base, d, c=c, blocks=blocks, rebuild=True)
                    seen |= w.seen
        assert across_eof > 0
    finally:
        shutil.rmtree(root, ignore_errors=True)
    direct_reads = (os.O_RDONLY, True) in seen
    direct_writes = any(dd and mode_ != os.O_RDONLY for mode_, dd in seen)
    assert (direct_reads, direct_writes) == (bool(mode & 1), bool(mode & 2)), (mode, sorted(seen), fs_type(where))


def _stale_ring_child(where):
    """Runs in a fresh process, so that the list of parked rings (at most four per process) starts empty and the ring
    each 0xFF call parks is the one the next call of its shape takes.  Every call here is RS(10,4) at a 4 KiB slot, one
    ring shape per slot count.  Asserts; exits non-zero on a mismatch."""
    from oracle import pyoracle as oracle

    import seaweedfs_b200 as swec
    import seaweedfs_b200._native  # noqa: F401  (swec._native)
    ec = swec.erasure_coding
    large, small = SWEEP_PAIR
    base = os.path.join(where, "r")

    def gen(dat):
        dat.tofile(base + ".dat")
        ec.generate_ec_files(base, math.gcd(large, small), large, small, ec.ECContext(10, 4))
        got = read_shards(base, 14)
        assert same(got, expected_shards(oracle, dat, 10, 4, large, small)), len(dat)
        return got

    for slots in (3, 2):
        set_option(swec, b"stage_slots", slots)
        # a tail row alone: its one item takes the first slot of the parked ring, which no earlier item of the call
        # has written, so only the zero fill past EOF keeps the 0xFF out of its padding; then a tail after several
        # items, and a verify and a repair whose last item is short
        for d in (3 * small + 17, large * 10 + 7 * small * 10 + 3 * small + 17):
            gen(random_dat(3 * large * 10, seed=0, fill=0xFF))          # whole 4 KiB items fill every slot with 0xFF
            clean = gen(random_dat(d, seed=d))
            assert ec.verify_ec_files(base) == (True, [0] * 4)
            size = len(clean[0])
            assert size % file_chunk(size, SWEEP_C)                     # the last item is short
            e = Edits(size)
            e.run(size - 20, size, 4)
            e.put(3, 12)
            damaged = e.apply(clean, seed=4)
            write_set(base, damaged)
            assert ec.repair_ec_damage(base) == {**do.locate(damaged, 10, 4), "ok": True}
            assert same(read_shards(base, 14), clean), (slots, d)
    print("RESULT ok")


@pytest.mark.gpu
def test_parked_ring_with_stale_bytes(cuda, swec, tmp_path):
    """A ring parked full of 0xFF by a call of the same shape: a tail row zero-padded past EOF, and a verify and a
    repair whose last item is short, must not see those bytes (in a child process: see _stale_ring_child)."""
    env = dict(os.environ, SWEC_FILE_CHUNK=str(SWEEP_C))
    for name in ("SWEC_NO_RING_CACHE", "SWEC_FILE_IO_PIECE", "SWEC_FILE_WRITE_PIECE", "SWEC_PIPE_STATS"):
        env.pop(name, None)
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; "
            f"import test_file_pipeline_exhaustive as t; t._stale_ring_child({str(tmp_path)!r})")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0 and "RESULT ok" in r.stdout, r.stderr[-4000:]


# ---------------------------------------------------------------------------------------------- GPU: the kernel switch


def _switch_child(where):
    """Runs in a fresh process with an empty SWEC_CACHE_DIR: a rebuild of shards 1, 5 and 12 (no compiled-in kernel)
    over 1,024 slots of 4 KiB, twice, under torch.profiler; between the calls, the background compile lands.  Prints
    RESULT <json>: the matrix-apply kernels of each call in launch order (None: no CUPTI) and whether the bytes match."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    import seaweedfs_b200 as swec
    import seaweedfs_b200._native  # noqa: F401  (swec._native)
    import test_kernel_variants as tkv
    ec = swec.erasure_coding
    L = swec.lib()
    set_option(swec, b"xt_variant", 1)                    # one kernel key, whatever the device's recent load
    torch.cuda.init()
    length, lost = 1024 * 4096, (1, 5, 12)
    clean = tdr.random_set(10, 4, length, seed=77)
    base = os.path.join(where, "k")
    write_set(base, clean)

    def compiles():
        c = C.c_uint64(0)
        swec._native.check(L.swec_jit_stats(C.byref(c), None, None, None))
        return c.value

    def run(b=base, want=clean):
        for i in lost:
            os.remove(b + ".ec%02d" % i)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ids = ec.rebuild_ec_files(b)
            torch.cuda.synchronize()
        events = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA), key=lambda e: e.time_range.start)
        kinds = [list(k) for k in map(tkv.kernel_id, [e.name for e in events]) if k is not None] if events else None
        return {"ids": ids, "kinds": kinds, "same": same(read_shards(b, 14), want)}

    c0 = compiles()
    first = run()
    t0 = time.time()
    while compiles() == c0 and time.time() - t0 < 300:
        time.sleep(0.05)
    compiled = compiles() > c0
    # the count goes up before the compiled library is loaded: rebuild a two-slot set of the same pattern until the
    # specialised kernel serves it (bounded; without CUPTI there is nothing to wait for)
    tiny_base, tiny = os.path.join(where, "t"), tdr.random_set(10, 4, 2 * 4096, seed=78)
    write_set(tiny_base, tiny)
    while compiled and time.time() - t0 < 300:
        kinds = run(tiny_base, tiny)["kinds"]
        if kinds is None or (kinds and all(k == ["swec_jit_flat"] for k in kinds)):
            break
        time.sleep(0.05)
    second = run()
    print("RESULT " + json.dumps({"first": first, "second": second, "compiled": compiled}))


@pytest.mark.gpu
def test_table_kernel_then_specialised_kernel(cuda, swec, tmp_path):
    env = dict(os.environ, SWEC_CACHE_DIR=str(tmp_path / "cubins"), SWEC_FILE_CHUNK="4096")
    env.pop("SWEC_FILE_JIT_WAIT", None)
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; "
            f"import test_file_pipeline_exhaustive as t; t._switch_child({str(tmp_path)!r})")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(next(ln for ln in r.stdout.splitlines() if ln.startswith("RESULT "))[7:])
    first, second = got["first"], got["second"]
    assert first["ids"] == second["ids"] == [1, 5, 12]
    assert first["same"] and second["same"] and got["compiled"]
    if first["kinds"] is None or second["kinds"] is None:
        import test_kernel_variants as tkv
        tkv.no_names("the rebuild's kernel switch")
        return
    assert first["kinds"][0][0] == "swec_table_kernel", first["kinds"][:4]
    print("specialised kernel within the first call: %s" % (["swec_jit_flat"] in first["kinds"]))
    assert second["kinds"] and all(k == ["swec_jit_flat"] for k in second["kinds"]), sorted(map(tuple, second["kinds"]))


# ---------------------------------------------------------------------------------------------- GPU: volume level


@pytest.mark.gpu
def test_volume_generate_reaches_the_pipeline(cuda, swec, oracle, tmp_path, capfd, knobs):
    """swec_ec_shards_generate runs the same pipeline at the default 1 GiB / 1 MiB geometry and 8 MiB slot."""
    ec = swec.erasure_coding
    knobs.delenv("SWEC_FILE_CHUNK", raising=False)
    dat, idx = tcd.needle_volume(seed=3, needles=300)
    base = str(tmp_path / "9")
    dat.tofile(base + ".dat")
    open(base + ".idx", "wb").write(idx)
    capfd.readouterr()
    ec.volume_ec_shards_generate(base)
    lines = [json.loads(x) for x in capfd.readouterr().err.splitlines() if x.startswith('{"pipe": "generate_ec_files"')]
    plan = item_plan(len(dat), 10, 1 << 30, 1 << 20, generate_chunk(1 << 30, 1 << 20, 8 << 20))
    assert [(x["items"], x["chunk"]) for x in lines] == [(len(plan), 8 << 20)]
    assert same(read_shards(base, 14), oracle.encode_dat_image(dat))
