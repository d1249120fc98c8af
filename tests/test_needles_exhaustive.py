"""The needle check (swec_check_needles_device, needles.cu with the walk of needle_format.h, and NeedleScrub of
ec_volume.cc behind swec_ec_volume_scrub_needles) at every Data alignment and length of the CRC's load paths, at every
16 KiB chunk seam, at every bound of the layout walk, and at every turn of the scrub's staging ring.

Each GPU case compares every output field of every record (status, range_index, data_size, crc_got, crc_want,
legacy_crc) with `expected`, which restates the check from needle_oracle.layout and the C CRC32-C of
tests/c/crc32c_oracle.c, and checks that the input fields (needle_id, offset, size, reserved) come back unchanged.
Tables are numpy arrays laid out like swec_needle_check, passed straight to the C call.

gpu, the CRC (needle_crc_kernel, needle_final_kernel):
  - version 1 records at every offset residue 0-15 x every Data length 0-260 (head 0-15 bytes, 0-3 steps of 64 bytes,
    0-15 words, a 0-3 byte tail), and the same image at base pointers shifted by 1-15 bytes;
  - Data lengths j*16384 + d, j = 1..5, d = -70..70, at alignments 0, 3, 4, 12 in versions 1 and 3, with random, all
    0x00, all 0xFF Data, Data with one interior chunk whose raw CRC is 0, and Data whose every full chunk's raw CRC is 0;
  - every record stored with its CRC, with CRC ^ 1 (BAD_CRC, not legacy) and with legacy_value(CRC) (BAD_CRC, legacy);
  - one version 1 record of Size 2^31 - 64, whole and with a byte flipped near its end.
gpu, the scan and the chunk-to-record search: 17 record counts from 1 to 65,537 x six patterns of records with and
without chunks (every record, every other, runs of 1,500 empty or failing records, only the first, only the last,
none); one record entered often enough for more than three grid-stride passes of the CRC kernel, between distinct ones.
gpu, the layout walk: versions 2 and 3, every flags value x name / mime lengths {0, 1, 254, 255} x pairs lengths
{0, 1, 0x100, 0xFFFF}, the body cut at every length up to its end + 4 (inside a 0xFFFF-byte pairs payload, only its
first 64 and last 4 cuts), every value of each byte of DataSize and of the name, mime and pairs lengths (on the
templates with every field flagged and pairs shorter than 0xFFFF), and index / header Size mismatches.
gpu, bounds (offsets -1, 0, dat_size, INT64_MAX, a record ending at dat_size and one byte past it, Size INT32_MAX,
with every byte past dat_size changed), stale output fields, user and default streams, four threads making the first
call of a fresh process.
gpu, NeedleScrub: a volume of 33,000 tiny records (slots full by count), then about 9 x 16 MiB of records (slots full
by bytes), a record of exactly one slot and one a slot + 8 bytes, walked to every slot of a 3- and a 2-slot ring after
it has wrapped, with damage on the first and last record of every slot turn; findings equal
test_needles.expected_findings in walk order.
cpu: record_layout compiled for the host against needle_oracle.layout on the layout corpus; the corpus reaches both
sides of every bound; the zero-CRC chunks; the needles.cu kernels in libswec.so are exactly the five this file runs."""
import ctypes as C
import functools
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import needle_oracle as no  # noqa: E402
import test_needles as tn  # noqa: E402

from oracle import rs_numpy as rn  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIB, GIB = 1 << 20, 1 << 30
CHUNK = 16384                                  # bytes of Data one lane of needle_crc_kernel checksums
SLOT_BYTES, SLOT_RECORDS = 16 * MIB, 16384     # one slot of NeedleScrub's staging ring
OK, SIZE_MISMATCH, OUT_OF_RANGE, BAD_CRC, OUTSIDE = 0, 1, 2, 3, 4
INT32_MAX, INT32_MIN, INT64_MAX = (1 << 31) - 1, -(1 << 31), (1 << 63) - 1
COOKIE = 0x0BADF00D

CHECK = np.dtype([("needle_id", "<u8"), ("offset", "<i8"), ("size", "<i4"), ("status", "<i4"), ("range_index", "<i4"),
                  ("data_size", "<u4"), ("crc_got", "<u4"), ("crc_want", "<u4"), ("legacy_crc", "<i4"),
                  ("reserved", "<i4")])
INPUTS = ("needle_id", "offset", "size", "reserved")
OUTPUTS = ("status", "range_index", "data_size", "crc_got", "crc_want", "legacy_crc")
KERNELS = {"needle_tables_kernel", "needle_parse_kernel", "needle_scan_kernel", "needle_crc_kernel",
           "needle_final_kernel"}


# ------------------------------------------------------------------------------------------ tables and the oracle


def table(offsets, sizes, ids=None):
    """Input fields of a check: `reserved` carries a pattern that must come back unchanged."""
    t = np.zeros(len(offsets), dtype=CHECK)
    t["offset"] = offsets
    t["size"] = sizes
    t["needle_id"] = np.arange(1, len(t) + 1, dtype=np.uint64) * 0x9E3779B1 if ids is None else ids
    t["reserved"] = (np.arange(len(t)) * 7919) ^ 0x5A5A5A5
    return t


def check_device(swec, ptr, dat_size, version, t, stream=None, stale=None):
    """swec_check_needles_device on a copy of `t` (output fields first set from `stale`, if given)."""
    from seaweedfs_b200._native import NeedleCheck, check
    out = t.copy()
    if stale is not None:
        for f in OUTPUTS:
            out[f] = stale[f]
    check(swec.lib().swec_check_needles_device(0, C.c_void_p(ptr), dat_size, version,
                                              C.cast(out.ctypes.data, C.POINTER(NeedleCheck)), len(out),
                                              None if stream is None else C.c_void_p(stream)))
    for f in INPUTS:
        assert np.array_equal(out[f], t[f]), f
    return out


def legacy(crc):
    crc = np.asarray(crc, dtype=np.uint64)
    return (((crc >> np.uint64(15)) | (crc << np.uint64(17))) + np.uint64(0xA282EAD8)) & np.uint64(0xFFFFFFFF)


def expected(img, dat_size, version, t):
    """The output fields Needle.ReadBytes gives each record of `t` (needle_oracle.layout, the C CRC32-C of Data), as
    the check reports them: OUTSIDE for a record not wholly inside [0, dat_size) (16 bytes for a negative Size),
    crc_want once the header Size matches, crc_got (the CRC of Data) and the legacy test only when there is Data."""
    want = t.copy()
    for f in OUTPUTS:
        want[f] = 0
    img = np.ascontiguousarray(img[:dat_size])
    at, length, rows = [], [], []
    for r, (off, size) in enumerate(zip(t["offset"].tolist(), t["size"].tolist())):
        need = 16 if size < 0 else no.actual_size(size, version)
        if off < 0 or off > dat_size or need > dat_size - off:
            want["status"][r] = OUTSIDE
            continue
        rec = img[off:off + need].tobytes()
        err, d_off, n = no.layout(rec, size, version)
        if err == "size mismatch":
            want["status"][r] = SIZE_MISMATCH
            continue
        want["crc_want"][r] = int.from_bytes(rec[16 + size:20 + size], "big")
        if err:
            want["status"][r] = OUT_OF_RANGE
            want["range_index"][r] = int(err.rsplit(" ", 1)[1])
            continue
        want["data_size"][r] = n
        if n:
            at.append(off + d_off)
            length.append(n)
            rows.append(r)
    if rows:
        rows = np.array(rows)
        got = no.ranges_crc32c(img, at, length)
        want["crc_got"][rows] = got
        bad = rows[got != want["crc_want"][rows]]
        want["status"][bad] = BAD_CRC
        want["legacy_crc"][bad] = legacy(want["crc_got"][bad]) == want["crc_want"][bad]
    return want


def assert_equal(got, want, what=""):
    for f in OUTPUTS:
        bad = np.nonzero(got[f] != want[f])[0]
        assert len(bad) == 0, (what, f, len(bad), got[bad[:4]], want[bad[:4]])


class Image:
    """A volume image built on the host, records placed at chosen offset residues mod 16."""

    def __init__(self, first=8):
        self.buf = bytearray(first)
        self.offsets, self.sizes = [], []

    def put(self, rec, size, residue=None):
        if residue is not None:
            self.buf += bytes((residue - len(self.buf)) % 16)
        self.offsets.append(len(self.buf))
        self.sizes.append(size)
        self.buf += rec
        return self.offsets[-1]

    def array(self, tail=0):
        return np.frombuffer(bytes(self.buf) + bytes(tail), dtype=np.uint8).copy()

    def table(self):
        return table(self.offsets, self.sizes)


def record(data, crc, version, nid=1):
    """A record of `data` with `crc` stored as its checksum (versions 2 and 3: no optional fields)."""
    return no.write_record(nid, data, version=version, cookie=COOKIE, checksum=int(crc), append_at_ns=nid)


def three_checksums(crc):
    """The stored forms every record is checked with: its CRC, the CRC ^ 1, and legacy_value(CRC)."""
    return (crc, crc ^ 1, no.legacy_value(crc))


def to_device(torch, img, shift=0):
    d = torch.empty(len(img) + shift, dtype=torch.uint8, device="cuda")
    d[shift:] = torch.from_numpy(img).cuda()
    return d


def check_stored_forms(got, n_data, crc):
    """Records of `n_data` bytes of Data stored with the three forms of `crc`, in that order, cycled."""
    for i, r in enumerate(got):
        if n_data[i] == 0:
            assert r["status"] == OK and r["crc_got"] == 0, i
        elif i % 3 == 0:
            assert r["status"] == OK and r["crc_got"] == r["crc_want"] == crc[i], i
        elif i % 3 == 1:
            assert (r["status"], r["crc_got"], r["legacy_crc"]) == (BAD_CRC, crc[i], 0), i
        else:
            assert (r["status"], r["crc_got"], r["legacy_crc"]) == (BAD_CRC, crc[i], 1), i


# ------------------------------------------------------------------------------------------ the zero-CRC chunks


def raw_crc(x) -> int:
    """The register of a CRC32-C started at 0 with no final XOR."""
    x = np.ascontiguousarray(x, dtype=np.uint8)
    return no.host_crc32c(x) ^ no.host_crc32c(np.zeros(len(x), dtype=np.uint8))


def zero_crc_chunk(rng):
    """16,384 bytes whose raw CRC is 0: 16,380 random bytes, then their raw CRC, little-endian."""
    head = rng.integers(0, 256, CHUNK - 4, dtype=np.uint8)
    return np.concatenate([head, np.frombuffer(raw_crc(head).to_bytes(4, "little"), dtype=np.uint8)])


SEAM_J, SEAM_D = range(1, 6), range(-70, 71)
SEAM_LONGEST = 5 * CHUNK + 70


@functools.lru_cache(maxsize=None)
def seam_contents():
    """Data long enough for every seam length, by name; each record takes a prefix."""
    rng = np.random.default_rng(0xC4C)
    chunks = -(-SEAM_LONGEST // CHUNK)
    random = rng.integers(0, 256, SEAM_LONGEST, dtype=np.uint8)
    one = random.copy()
    one[CHUNK:2 * CHUNK] = zero_crc_chunk(rng)
    every = np.concatenate([zero_crc_chunk(rng) for _ in range(chunks)])[:SEAM_LONGEST]
    return {"random": random, "zeros": np.zeros(SEAM_LONGEST, dtype=np.uint8),
            "ones": np.full(SEAM_LONGEST, 0xFF, dtype=np.uint8), "one zero-CRC chunk": one,
            "every full chunk zero-CRC": every}


def seam_lengths():
    return [j * CHUNK + d for j in SEAM_J for d in SEAM_D]


# ------------------------------------------------------------------------------------------ the layout corpus

FIELD_LENGTHS = (0, 1, 254, 255)
PAIRS_LENGTHS = (0, 1, 0x100, 0xFFFF)
LAYOUT_DATA = 5


def template_body(rng, flags, name, mime, pairs):
    """A v2/v3 body with LAYOUT_DATA bytes of Data, `flags` as stored, and the fields `flags` names."""
    out = bytearray(LAYOUT_DATA.to_bytes(4, "big")) + rng.integers(0, 256, LAYOUT_DATA, dtype=np.uint8).tobytes()
    out.append(flags)
    if flags & no.FLAG_NAME:
        out += bytes([name]) + rng.integers(0, 256, name, dtype=np.uint8).tobytes()
    if flags & no.FLAG_MIME:
        out += bytes([mime]) + rng.integers(0, 256, mime, dtype=np.uint8).tobytes()
    if flags & no.FLAG_LAST_MODIFIED:
        out += (1_700_000_000).to_bytes(5, "big")
    if flags & no.FLAG_TTL:
        out += b"\x05\x03"
    pairs_at = len(out) + 2
    if flags & no.FLAG_PAIRS:
        out += pairs.to_bytes(2, "big") + rng.integers(0, 256, pairs, dtype=np.uint8).tobytes()
    return bytes(out), pairs_at


def templates():
    """Every flags value with the name / mime / pairs lengths of each rotation j (name FIELD_LENGTHS[j], mime
    FIELD_LENGTHS[j + 1], pairs PAIRS_LENGTHS[j + 2]), and all 64 length combinations with every field flagged."""
    keys = set()
    for flags in range(256):
        for j in range(4):
            keys.add((flags, FIELD_LENGTHS[j] if flags & no.FLAG_NAME else 0,
                      FIELD_LENGTHS[(j + 1) % 4] if flags & no.FLAG_MIME else 0,
                      PAIRS_LENGTHS[(j + 2) % 4] if flags & no.FLAG_PAIRS else 0))
    every = 0x3E
    full = {(every, a, b, c) for a in FIELD_LENGTHS for b in FIELD_LENGTHS for c in PAIRS_LENGTHS}
    return sorted(keys | full), full


def cuts(body_len, pairs_at):
    """Every cut 0 .. body + 4, except inside a 0xFFFF-byte pairs payload: its first 64 cuts and its last 4."""
    if body_len <= 4096:
        return range(body_len + 5)
    return list(range(pairs_at + 64)) + list(range(body_len - 4, body_len + 5))


def header(size, nid=1):
    return COOKIE.to_bytes(4, "big") + nid.to_bytes(8, "big") + (size & 0xFFFFFFFF).to_bytes(4, "big")


@functools.lru_cache(maxsize=None)
def layout_corpus(version):
    """(image, table, kind, cut_of) of the layout sweep: kind 0 for a cut (its template and cut in `cut_of`), 1 for a
    byte of a length field set to a value, 2 for a Size mismatch.  A cut record is its header with Size = the cut,
    then the template's body and real checksum up to 4 bytes past the cut: those 4 bytes are what the walk reads as
    the checksum, as on disk."""
    rng = np.random.default_rng(0x1A70 + version)
    keys, full = templates()
    img = Image()
    kinds, cut_of = [], []

    def lay(size, stored, index_size, kind, where):
        rec = header(size) + stored
        rec += bytes(max(no.actual_size(max(size, 0), version), len(rec) + 7) // 8 * 8 - len(rec))
        img.put(rec, index_size)
        kinds.append(kind)
        cut_of.append(where)

    for t, key in enumerate(keys):
        body, pairs_at = template_body(rng, *key)
        n = len(body)
        whole = body + no.host_crc32c(body[4:4 + LAYOUT_DATA]).to_bytes(4, "big")
        for cut in cuts(n, pairs_at):
            lay(cut, whole[:cut + 4], cut, 0, (t, cut))
        for s in (n + 1, n - 1, -1, INT32_MIN):          # the index Size disagrees with the header
            lay(n, whole, s, 2, (t, -1))
        lay(-5, whole, -5, 2, (t, -1))                    # a negative header Size
        if key in full and key[3] != 0xFFFF:
            name_at = 4 + LAYOUT_DATA + 1
            mime_at = name_at + 1 + key[1]
            for at in (0, 1, 2, 3, name_at, mime_at, pairs_at - 2, pairs_at - 1):
                b = bytearray(whole)
                for v in range(256):
                    b[at] = v
                    lay(n, bytes(b), n, 1, (t, -1))
    t = img.table()
    return img.array(), t, np.array(kinds), cut_of


def host_layout_library(tmp_path):
    src = tmp_path / "layout.cc"
    src.write_text('#include "%s"\n' % os.path.join(ROOT, "seaweedfs_b200", "csrc", "needle_format.h") + r'''
extern "C" void layout_all(const uint8_t* img, const int64_t* off, const int32_t* size, int n, int version,
                           int64_t* out) {
    for (int i = 0; i < n; i++) {
        const swec::RecordLayout l = swec::record_layout(img + off[i], size[i], version);
        int64_t* o = out + 5 * int64_t(i);
        o[0] = l.status, o[1] = l.range_index, o[2] = l.data_size, o[3] = l.data_offset, o[4] = l.crc_want;
    }
}
''')
    so = str(tmp_path / "liblayout.so")
    subprocess.run(["c++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, str(src)], check=True)
    L = C.CDLL(so)
    L.layout_all.argtypes = [C.c_void_p] * 3 + [C.c_int, C.c_int, C.c_void_p]
    return L


# ------------------------------------------------------------------------------------------ CPU


def test_check_dtype_matches_the_binding():
    from seaweedfs_b200._native import NeedleCheck
    assert CHECK.itemsize == C.sizeof(NeedleCheck)
    assert all(CHECK.fields[f][1] == getattr(NeedleCheck, f).offset for f, _ in NeedleCheck._fields_)


def test_zero_crc_chunks():
    """The recipe's chunks really have raw CRC 0, by the C CRC32-C; the one-chunk content's neighbours do not."""
    c = seam_contents()
    for name in ("one zero-CRC chunk", "every full chunk zero-CRC"):
        raws = [raw_crc(c[name][i:i + CHUNK]) for i in range(0, SEAM_LONGEST - CHUNK + 1, CHUNK)]
        assert len(raws) == 5
        if name == "one zero-CRC chunk":
            assert raws[1] == 0 and all(raws[i] != 0 for i in (0, 2, 3, 4))
        else:
            assert raws == [0] * 5 and raw_crc(c[name][5 * CHUNK:]) != 0
    assert raw_crc(c["zeros"][:CHUNK]) == 0 and raw_crc(c["ones"][:CHUNK]) != 0
    # a whole record of zero-CRC chunks still has a CRC32-C that is not zero (the init and final XOR)
    assert no.host_crc32c(c["every full chunk zero-CRC"][:2 * CHUNK]) == no.host_crc32c(np.zeros(2 * CHUNK, np.uint8))


@pytest.mark.parametrize("version", [2, 3])
def test_layout_corpus_reaches_both_sides_of_every_bound(version):
    """For each range_index 1-7 some template fails it at a cut and passes it one byte later; every flags value is
    walked; the byte sweeps and mismatches give OUT_OF_RANGE 1-3, 6-7 and SIZE_MISMATCH."""
    img, t, kinds, cut_of = layout_corpus(version)
    want = expected(img, len(img), version, t)
    at = {w: r for r, w in enumerate(cut_of) if w[1] >= 0}
    sides = {i: [0, 0] for i in range(1, 8)}
    for (tpl, cut), r in at.items():
        i = want["range_index"][r]
        if i and (tpl, cut + 1) in at:
            sides[i][0] += 1
            sides[i][1] += want["range_index"][at[(tpl, cut + 1)]] != i
    assert all(a > 0 and b > 0 for a, b in sides.values()), sides
    assert {int(x) for x in want["range_index"][kinds == 1]} >= {0, 1, 2, 3, 6, 7}
    assert set(want["status"][kinds == 2].tolist()) == {SIZE_MISMATCH}
    assert set(want["status"][kinds == 0].tolist()) == {OK, OUT_OF_RANGE, BAD_CRC}
    flags_seen = {img[o + 16 + 4 + LAYOUT_DATA] for o, k in zip(t["offset"], kinds) if k == 0}
    assert len(flags_seen) == 256


@pytest.mark.parametrize("version", [2, 3])
def test_host_record_layout_equals_the_oracle(tmp_path, version):
    """needle_format.h's record_layout, compiled for the host, against needle_oracle.layout on the layout corpus."""
    L = host_layout_library(tmp_path)
    img, t, _, _ = layout_corpus(version)
    want = expected(img, len(img), version, t)
    inside = want["status"] != OUTSIDE       # the walk's precondition: the record's bytes are all there
    t, want = t[inside], want[inside]
    out = np.zeros((len(t), 5), dtype=np.int64)
    off, size = np.ascontiguousarray(t["offset"]), np.ascontiguousarray(t["size"])
    L.layout_all(img.ctypes.data, off.ctypes.data, size.ctypes.data, len(t), version, out.ctypes.data)
    status = np.where(want["status"] == BAD_CRC, OK, want["status"])
    assert np.array_equal(out[:, 0], status)
    assert np.array_equal(out[:, 1], want["range_index"])
    assert np.array_equal(out[:, 2], want["data_size"])
    assert np.array_equal(out[:, 4], want["crc_want"])
    ok = status == OK
    assert np.array_equal(out[ok, 3], np.where(t["size"][ok] > 0, 20, 16))
    assert inside.sum() > len(inside) - 10


def test_needle_kernels_in_the_library_are_the_five(swec):
    """The __global__ functions of needles.cu in libswec.so are exactly the five this file runs."""
    from seaweedfs_b200 import _native
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("no CUDA toolkit")
    out = subprocess.run([cuobjdump, "-symbols", _native.library_path()], capture_output=True, text=True,
                         check=True).stdout
    syms = [ln.split()[-1] for ln in out.splitlines() if "STT_FUNC" in ln and "STO_ENTRY" in ln and "_needles_cu_" in ln]
    names = [re.search(r"\d(needle_[a-z]+_kernel)E", s)[1] for s in syms]
    assert len(names) == len(set(names)) and set(names) == KERNELS, syms


# ------------------------------------------------------------------------------------------ GPU: the CRC paths


@pytest.mark.gpu
def test_every_alignment_and_short_length(cuda, swec):
    """Version 1 records at every offset residue 0-15 x Data lengths 0-260, each stored with its three checksum
    forms; then the same image at base pointers shifted by 1 to 15 bytes."""
    torch = cuda
    rng = np.random.default_rng(0xA1)
    img = Image()
    crcs, lens = [], []
    for residue in range(16):
        for n in range(261):
            data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            crc = no.host_crc32c(data)
            for stored in three_checksums(crc):
                img.put(record(data, stored, 1), n, residue)
                crcs.append(crc)
                lens.append(n)
    host, t = img.array(), img.table()
    assert {int(o + 16) % 16 for o in t["offset"]} == set(range(16))
    want = expected(host, len(host), 1, t)
    for shift in range(16):
        d = to_device(torch, host, shift)
        got = check_device(swec, d.data_ptr() + shift, len(host), 1, t)
        assert_equal(got, want, shift)
    check_stored_forms(got, lens, crcs)


@pytest.mark.gpu
@pytest.mark.parametrize("content", ["random", "zeros", "ones", "one zero-CRC chunk", "every full chunk zero-CRC"])
def test_chunk_seams(cuda, swec, content):
    """Data lengths j*16384 + d (j = 1..5, d = -70..70) at alignments 0, 3, 4, 12, versions 1 and 3, each stored with
    its three checksum forms."""
    torch = cuda
    source = seam_contents()[content]
    crc = {n: no.host_crc32c(source[:n]) for n in seam_lengths()}
    for version in (1, 3):
        img = Image()
        crcs, lens = [], []
        data_at = 16 if version == 1 else 20
        for align in (0, 3, 4, 12):
            for n in seam_lengths():
                data = source[:n].tobytes()
                for stored in three_checksums(crc[n]):
                    img.put(record(data, stored, version), n + (0 if version == 1 else 5), (align - data_at) % 16)
                    crcs.append(crc[n])
                    lens.append(n)
        host, t = img.array(), img.table()
        assert {int(o + data_at) % 16 for o in t["offset"]} == {0, 3, 4, 12}
        d = to_device(torch, host)
        got = check_device(swec, d.data_ptr(), len(host), version, t)
        assert_equal(got, expected(host, len(host), version, t), version)
        check_stored_forms(got, lens, crcs)
        del d


@pytest.mark.gpu
def test_largest_record(cuda, swec):
    """One version 1 record of Size 2^31 - 64, Data from the seeded stream: OK with its CRC, BAD_CRC with the oracle's
    CRC once a byte near its end is flipped."""
    torch = cuda
    size = (1 << 31) - 64
    total = 8 + no.actual_size(size, 1)
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < total + (2 << 30):
        pytest.skip(f"needs {total + (2 << 30)} B of free HBM, {free} free")
    d = torch.empty(total, dtype=torch.uint8, device="cuda")
    try:
        swec._native.check(swec.lib().swec_synth_fill_device(0, d.data_ptr(), 0, total, tn.SEED, None))
        d[8:24] = torch.frombuffer(bytearray(header(size, 77)), dtype=torch.uint8).cuda()
        host = d.cpu().numpy()
        crc = no.host_crc32c(host[24:24 + size])
        tail = torch.frombuffer(bytearray(crc.to_bytes(4, "big")), dtype=torch.uint8).cuda()
        d[24 + size:28 + size] = tail
        host[24 + size:28 + size] = np.frombuffer(crc.to_bytes(4, "big"), dtype=np.uint8)
        t = table([8], [size])
        got = check_device(swec, d.data_ptr(), total, 1, t)
        assert (got["status"][0], got["crc_got"][0], got["data_size"][0]) == (OK, crc, size)
        assert_equal(got, expected(host, total, 1, t))
        x = 24 + size - 1000
        d[x] ^= 0x10
        host[x] ^= 0x10
        got = check_device(swec, d.data_ptr(), total, 1, t)
        assert (got["status"][0], got["crc_want"][0], got["legacy_crc"][0]) == (BAD_CRC, crc, 0)
        assert_equal(got, expected(host, total, 1, t))
        assert got["crc_got"][0] == no.host_crc32c(host[24:24 + size])
    finally:
        del d
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ GPU: scan and search

COUNTS = [1, 2, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049, 4097, 16384, 65537]
PATTERNS = ["every", "every other", "runs of 1500", "first only", "last only", "none"]


@functools.lru_cache(maxsize=None)
def pool():
    """A version 1 image of 61 distinct records of 1 to 4 chunks (every fifth stored with a wrong CRC), one empty
    record and one whose index Size disagrees with its header.  Returns (image, table of the pool)."""
    rng = np.random.default_rng(0x5CA)
    img = Image()
    for i in range(61):
        n = int(rng.integers(1, 4 * CHUNK + 1))
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        crc = no.host_crc32c(data)
        img.put(record(data, crc ^ (i % 5 == 0), 1, nid=i + 1), n)
    img.put(record(b"", 0, 1, nid=100), 0)
    img.put(record(b"abc", no.host_crc32c(b"abc"), 1, nid=101), 2)
    return img.array(), img.table()


def pattern_rows(pattern, n, data=61, empty=61, failing=62):
    """Pool rows of n entries: consecutive entries with Data point at different records."""
    cyc = np.arange(n) % data
    quiet = np.where(np.arange(n) % 2 == 0, empty, failing)
    if pattern == "every":
        return cyc
    if pattern == "every other":
        return np.where(np.arange(n) % 2 == 0, (np.arange(n) // 2) % data, empty)
    if pattern == "runs of 1500":
        i = np.arange(n)
        run = (i // 1501) % 2
        return np.where(i % 1501 == 0, (i // 1501) % data, np.where(run == 0, empty, failing))
    if pattern == "first only":
        return np.where(np.arange(n) == 0, 0, quiet)
    if pattern == "last only":
        return np.where(np.arange(n) == n - 1, 1, quiet)
    return quiet


@pytest.mark.gpu
def test_scan_and_search_at_every_count_and_pattern(cuda, swec):
    torch = cuda
    host, pt = pool()
    pwant = expected(host, len(host), 1, pt)
    assert pwant["status"][61] == OK and pwant["data_size"][61] == 0 and pwant["status"][62] == SIZE_MISMATCH
    assert set(pwant["status"][:61].tolist()) == {OK, BAD_CRC}
    d = to_device(torch, host)
    for n in COUNTS:
        for pattern in PATTERNS:
            rows = pattern_rows(pattern, n)
            t = table(pt["offset"][rows], pt["size"][rows])
            want = pwant[rows].copy()
            for f in INPUTS:
                want[f] = t[f]
            got = check_device(swec, d.data_ptr(), len(host), 1, t)
            assert_equal(got, want, (n, pattern))


@pytest.mark.gpu
def test_several_grid_stride_passes(cuda, swec):
    """One 1 MiB record (64 chunks) entered often enough for more than 3 x SMs x 1024 chunks, with distinct records,
    some damaged, between its entries."""
    torch = cuda
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(0x6A1D)
    img = Image()
    data = rng.integers(0, 256, MIB, dtype=np.uint8).tobytes()
    img.put(record(data, no.host_crc32c(data), 1), MIB)
    for i in range(40):
        n = int(rng.integers(0, 3 * CHUNK))
        small = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        img.put(record(small, no.host_crc32c(small) ^ (i % 3 == 0), 1, nid=i + 2), n if i % 7 else n + 1)
    host, pt = img.array(), img.table()
    entries = 3 * sms * 1024 // 64 + 300
    rows = np.where(np.arange(entries) % 50 == 7, 1 + np.arange(entries) % 40, 0)
    t = table(pt["offset"][rows], pt["size"][rows])
    want = expected(host, len(host), 1, pt)[rows].copy()
    for f in INPUTS:
        want[f] = t[f]
    assert int(((want["data_size"].astype(np.int64) + CHUNK - 1) // CHUNK).sum()) > 3 * sms * 1024
    assert set(want["status"].tolist()) == {OK, BAD_CRC, SIZE_MISMATCH}
    d = to_device(torch, host)
    assert_equal(check_device(swec, d.data_ptr(), len(host), 1, t), want)


# ------------------------------------------------------------------------------------------ GPU: the layout walk


@pytest.mark.gpu
@pytest.mark.parametrize("version", [2, 3])
def test_layout_walk(cuda, swec, version):
    torch = cuda
    img, t, _, _ = layout_corpus(version)
    d = to_device(torch, img)
    got = check_device(swec, d.data_ptr(), len(img), version, t)
    assert_equal(got, expected(img, len(img), version, t), version)
    assert set(got["range_index"].tolist()) == set(range(8))


# ------------------------------------------------------------------------------------------ GPU: bounds, stale, streams


def bounds_case():
    """Records inside, at and past the end of the image; returns (image, dat_size, table)."""
    rng = np.random.default_rng(0xB0)
    img = Image()
    for n in (0, 1, 100, 5000):
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        img.put(record(data, no.host_crc32c(data), 3, nid=n + 1), n + 5, 3)
    data = rng.integers(0, 256, 333, dtype=np.uint8).tobytes()
    last = img.put(record(data, no.host_crc32c(data), 3, nid=9), 338)
    dat_size = len(img.buf)
    offs = img.offsets + [-1, 0, dat_size, INT64_MAX, dat_size - 16, dat_size - 15, img.offsets[2], img.offsets[2],
                          img.offsets[1], last]
    sizes = img.sizes + [0, 0, 0, 0, -1, -1, INT32_MAX, INT32_MIN, -1, 338]
    return img.array(), dat_size, table(offs, sizes), last


@pytest.mark.gpu
def test_bounds_and_bytes_past_the_image(cuda, swec):
    """A record ending exactly at dat_size is checked and one byte short of it is OUTSIDE; offsets -1, 0, dat_size,
    INT64_MAX, Size INT32_MAX / INT32_MIN / -1; then every byte of the allocation past dat_size changed."""
    torch = cuda
    host, dat_size, t, last = bounds_case()
    tail = 4096
    d = to_device(torch, np.concatenate([host, np.zeros(tail, np.uint8)]))
    for size in (dat_size, dat_size - 1):
        want = expected(host, size, 3, t)
        rows = np.nonzero(t["offset"] == last)[0]
        assert set(want["status"][rows].tolist()) == ({OK} if size == dat_size else {OUTSIDE})
        for fill in (0x00, 0xFF, 0xA5, -1):
            past = d[size:]
            if fill < 0:
                past.copy_(torch.randint(0, 256, past.shape, dtype=torch.uint8, device="cuda"))
            else:
                past.fill_(fill)
            assert_equal(check_device(swec, d.data_ptr(), size, 3, t), want, (size, fill))
    assert set(want["status"].tolist()) == {OK, SIZE_MISMATCH, OUTSIDE}


@pytest.mark.gpu
def test_stale_fields_and_streams(cuda, swec):
    """Garbage in the output fields never reaches the result; the same call on a user stream and on the default
    stream, twice each, gives the same results."""
    torch = cuda
    host, pt = pool()
    rows = pattern_rows("runs of 1500", 5000)
    t = table(pt["offset"][rows], pt["size"][rows])
    d = to_device(torch, host)
    clean = check_device(swec, d.data_ptr(), len(host), 1, t)
    want = expected(host, len(host), 1, pt)[rows]
    for f in INPUTS:
        want[f] = t[f]
    assert_equal(clean, want)
    rng = np.random.default_rng(3)
    stale = np.zeros(len(t), dtype=CHECK)
    for f in OUTPUTS:
        stale[f] = rng.integers(0, 1 << 31, len(t)).astype(stale[f].dtype)
    assert_equal(check_device(swec, d.data_ptr(), len(host), 1, t, stale=stale), clean, "stale")
    s = torch.cuda.Stream()
    for stream in (s.cuda_stream, None, s.cuda_stream, None):
        assert_equal(check_device(swec, d.data_ptr(), len(host), 1, t, stream=stream), clean, stream)


THREADS_CHILD = r"""
import json, sys, threading
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
import numpy as np, torch
import seaweedfs_b200 as swec
import test_needles_exhaustive as tne
host, pt = tne.pool()
rows = tne.pattern_rows("every other", 3000)
t = tne.table(pt["offset"][rows], pt["size"][rows])
d = torch.from_numpy(host).cuda()
streams = [torch.cuda.Stream() for _ in range(4)]
torch.cuda.synchronize()
gate, out, errors = threading.Barrier(4), [None] * 4, []
def run(i):
    try:
        gate.wait()
        out[i] = tne.check_device(swec, d.data_ptr(), len(host), 1, t, stream=streams[i].cuda_stream)
    except Exception as e:
        errors.append(repr(e))
ths = [threading.Thread(target=run, args=(i,)) for i in range(4)]
[x.start() for x in ths]
[x.join() for x in ths]
want = tne.expected(host, len(host), 1, pt)[rows]
print(json.dumps({"errors": errors, "same": [bool(all(np.array_equal(o[f], want[f]) for f in tne.OUTPUTS))
                                            for o in out if o is not None]}))
"""


@pytest.mark.gpu
def test_first_calls_from_four_threads(cuda, swec):
    """Four threads of a fresh process make their first call at once, each on its own stream, while the per-device
    tables are not built yet."""
    r = subprocess.run([sys.executable, "-c", THREADS_CHILD, ROOT, os.path.dirname(os.path.abspath(__file__))],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert got == {"errors": [], "same": [True] * 4}


# ------------------------------------------------------------------------------------------ GPU: NeedleScrub


def slot_turns(actual_sizes):
    """The staging-slot turn (0, 1, ...) in which NeedleScrub checks each record of a walk, or -1 for a record larger
    than a slot (checked from a buffer of its own): a record starts a new turn when its bytes do not fit in what is
    left of the slot, or the slot already holds 16,384 records.  Turn t uses slot t % stage_slots."""
    out, turn, used, count = [], 0, 0, 0
    for n in actual_sizes:
        if n > SLOT_BYTES:
            out.append(-1)
            continue
        if count and (used + n > SLOT_BYTES or count == SLOT_RECORDS):
            turn, used, count = turn + 1, 0, 0
        out.append(turn)
        used += (n + 7) & ~7
        count += 1
    return np.array(out)


def scrub_data_lengths(rng):
    """Data lengths in walk order: 33,000 tiny records, then records of 4 KiB to 3 MiB for about 9 slots, with one
    record of exactly one slot and one of a slot + 8 bytes about halfway."""
    tiny = [0 if i % 11 == 0 else int(rng.integers(1, 40)) for i in range(33_000)]
    body = [int(np.exp(rng.uniform(np.log(4096), np.log(3 * MIB)))) for _ in range(300)]
    exact, over = SLOT_BYTES - 37, SLOT_BYTES - 29   # v3, no optional fields: actual sizes 16 MiB and 16 MiB + 8
    assert no.actual_size(exact + 5, 3) == SLOT_BYTES and no.actual_size(over + 5, 3) == SLOT_BYTES + 8
    return tiny + body[:150] + [exact, over] + body[150:]


def scrub_volume(oracle, tmp_path, rng):
    """A v3 volume of scrub_data_lengths' records laid down as EC shards.  Returns (base, dat, entries)."""
    lengths = scrub_data_lengths(rng)
    source = rng.integers(0, 256, max(lengths) + 1024, dtype=np.uint8)
    parts, idx, entries, pos = [bytes([3, 0, 0, 0, 0, 0, 0, 0])], [], [], 8
    for i, n in enumerate(lengths):
        start = int(rng.integers(0, 1024))
        data = source[start:start + n]
        rec = no.write_record(1000 + i, data.tobytes(), version=3, checksum=no.host_crc32c(data), append_at_ns=i)
        size = int.from_bytes(rec[12:16], "big")
        entries.append((1000 + i, pos, size))
        idx.append(rn._entry(1000 + i, pos // 8, size))
        parts.append(rec)
        pos += len(rec)
    dat = np.frombuffer(b"".join(parts), dtype=np.uint8).copy()
    base = str(tmp_path / "9")
    for i, s in enumerate(oracle.encode_dat_image(dat)):
        s.tofile(base + ".ec%02d" % i)
    open(base + ".ecx", "wb").write(rn.sorted_ecx_from_idx(b"".join(idx)))
    json.dump({"version": 3, "datFileSize": str(len(dat)), "ecShardConfig": {"dataShards": 10, "parityShards": 4}},
              open(base + ".vif", "w"))
    return base, dat, entries


def damage(base, dat, entry, rng):
    """A flipped Data byte, or the header Size when the record has no Data."""
    k, off, size = entry
    n = int.from_bytes(dat[off + 16:off + 20].tobytes(), "big")
    x = off + 20 + int(rng.integers(0, n)) if n else off + 15
    dat[x] ^= 0x40 if n else 0x08
    tn.poke_shard(base, x, int(dat[x]))


@pytest.mark.gpu
def test_scrub_slot_turns(cuda, swec, oracle, tmp_path):
    """Walks that end on every slot of a 3- and a 2-slot ring after it has wrapped, and the whole volume; findings and
    (entries, broken) as test_needles.expected_findings and scrub_local say."""
    ec = swec.erasure_coding
    vid = 9
    rng = np.random.default_rng(0x5107)
    base, dat, entries = scrub_volume(oracle, tmp_path, rng)
    turns = slot_turns([no.actual_size(s, 3) for _, _, s in entries])
    last = int(turns.max())
    firsts = [int(np.nonzero(turns == t)[0][0]) for t in range(last + 1)]
    lasts = [int(np.nonzero(turns == t)[0][-1]) for t in range(last + 1)]
    # coverage of the ring: two turns full by count, the rest by bytes, a one-record turn of a whole slot, and a
    # record larger than a slot between two full turns
    assert lasts[0] - firsts[0] + 1 == lasts[1] - firsts[1] + 1 == SLOT_RECORDS and last >= 9
    big = int(np.nonzero(turns == -1)[0][0])
    assert firsts[turns[big - 1]] == big - 1 and turns[big + 1] == turns[big - 1] + 1
    for r in sorted(set(firsts) | set(lasts) | {big}):
        damage(base, dat, entries[r], rng)

    def walk(n, slots):
        ib = str(tmp_path / f"w{n}")
        open(ib + ".ecx", "wb").write(b"".join(rn._entry(k, off // 8, s) for k, off, s in entries[:n]))
        vol = ec.EcVolume(base, ib, device=0)
        try:
            count, broken, findings = vol.scrub_needles(vid)
            assert (count, broken) == vol.scrub_local()[:2] == (n, [])
        finally:
            vol.close()
        assert findings == tn.expected_findings(dat, entries[:n], vid), (n, slots)
        return findings

    L = swec.lib()
    try:
        for slots in (3, 2):
            swec._native.check(L.swec_set_option(b"stage_slots", slots))
            ends = [t for t in range(2 * slots, last + 1)][:slots]
            assert sorted(t % slots for t in ends) == list(range(slots))
            for t in ends:
                assert len(walk(lasts[t] + 1, slots)) >= t + 1
            walk(len(entries), slots)
    finally:
        swec._native.check(L.swec_set_option(b"stage_slots", 3))
