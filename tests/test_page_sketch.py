"""Page sketches of EC shards, and damage located from the sketches of a whole set (include/swec.h,
SWEC_PAGE_SKETCH_VERSION): swec_page_sketch_device, swec_page_sketch_file and swec_locate_sketch_damage.

CPU: a numpy sketch oracle (pyoracle.synth weights, rs_numpy's GF tables) against a literal per-byte loop; linearity and
the codeword property of sketches; a page-decode oracle built on damage_oracle that meets the per-page guarantee for
every damaged shard set of RS(3,2) and RS(6,3); the argument rules of the three calls on a device-less encoder.
GPU: device and file sketches bit-exact against the oracle; the page decode against the page oracle on a damage corpus
and against swec_locate_ec_damage's ranges; and the scrub of a set whose shard files each sit in a directory of their
own, repaired by fetching only the flagged pages.
"""
import ctypes as C
import itertools
import os
import re

import numpy as np
import pytest

import damage_oracle as do
from oracle import rs_numpy as rn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGE = 4096
MASK64 = (1 << 64) - 1
CODES = [(10, 4), (6, 3), (20, 12), (3, 2)]


# ---------------------------------------------------------------------------------------------------------- oracles

def sketch(pyoracle, c: np.ndarray, seed: int, first_column: int = 0) -> np.ndarray:
    """The sketch of shard bytes c whose first byte is shard offset first_column: uint64 per 4 KiB page."""
    n = len(c)
    if n == 0:
        return np.zeros(0, dtype=np.uint64)
    w = pyoracle.synth(8 * first_column, 8 * n, seed).reshape(n, 8)   # w_l(x): byte l of word x of the stream
    prod = rn.MUL[w, c[:, None]]
    return np.ascontiguousarray(np.bitwise_xor.reduceat(prod, np.arange(0, n, PAGE), axis=0)).view("<u8").ravel()


def splitmix(seed: int, x: int) -> int:
    z = (seed + (x + 1) * 0x9E3779B97F4A7C15) & MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
    return z ^ (z >> 31)


def sketch_loop(c: bytes, seed: int, first_column: int = 0) -> list[int]:
    """The definition, one byte at a time."""
    out = []
    for g in range(0, len(c), PAGE):
        acc = [0] * 8
        for x in range(g, min(g + PAGE, len(c))):
            w = splitmix(seed, first_column + x)
            for lb in range(8):
                acc[lb] ^= rn.gf_mul((w >> (8 * lb)) & 0xFF, c[x])
        out.append(sum(a << (8 * lb) for lb, a in enumerate(acc)))
    return out


def page_oracle(sketches, k: int, m: int, radius: int) -> list[tuple[int, int, bool]]:
    """(page, blamed mask, uncorrectable) of every flagged page: damage_oracle decodes every byte of the sketches as a
    column, and a page is blamed on the union of its columns' shards unless a column is uncorrectable or the union
    exceeds the radius."""
    shards = [np.ascontiguousarray(s, dtype="<u8").view(np.uint8) for s in sketches]
    cols, a, b, _, _, ids = do.decode_columns(shards, k, m, radius)
    pages = {}
    for c, x, y in zip(cols.tolist(), a.tolist(), b.tolist()):
        mask, bad = pages.get(c // 8, (0, False))
        if x < 0:
            bad = True
        else:
            mask |= 1 << int(ids[x])
            if y >= 0:
                mask |= 1 << int(ids[y])
        pages[c // 8] = (mask, bad)
    out = []
    for g in sorted(pages):
        mask, bad = pages[g]
        bad = bad or bin(mask).count("1") > radius
        out.append((g, 0 if bad else mask, bad))
    return out


def clean_set(k, m, n, seed):
    rng = np.random.default_rng(seed)
    data = [rng.integers(0, 256, n, dtype=np.uint8) for _ in range(k)]
    return data + rn.encode(k, m, data)


def mask_of(ids):
    return sum(1 << i for i in ids)


# ---------------------------------------------------------------------------------------------------------- CPU

def test_version_is_in_the_header():
    header = open(os.path.join(ROOT, "include", "swec.h")).read()
    assert re.search(r"^#define SWEC_PAGE_SKETCH_VERSION 1\b", header, re.M)


@pytest.mark.parametrize("n,first_column,seed", [(1, 0, 0), (17, 4096, MASK64), (4096 + 300, 1 << 32, 0x1234567890ABCDEF),
                                                 (2 * 4096, 3 * (1 << 30) - 4096, 7)])
def test_numpy_oracle_is_the_definition(oracle, n, first_column, seed):
    c = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8)
    assert sketch(oracle, c, seed, first_column).tolist() == sketch_loop(c.tobytes(), seed, first_column)


@pytest.mark.parametrize("k,m", CODES)
def test_linearity_and_codewords(oracle, k, m):
    n = 3 * PAGE + 123
    seed = 0xC0FFEE + k
    shards = clean_set(k, m, n, k * 100 + m)
    sk = [sketch(oracle, s, seed) for s in shards]
    as_bytes = [s.view(np.uint8) for s in sk]
    # the sketch bytes of a clean set are a codeword of the same code, column by column
    parity = rn.apply_rows(rn.build_matrix(k, k + m)[k:], as_bytes[:k])
    for p in range(m):
        assert (parity[p] == as_bytes[k + p]).all()
    # σ(a⊗c ⊕ b⊗c') = a⊗σ(c) ⊕ b⊗σ(c')
    rng = np.random.default_rng(k)
    c1, c2 = shards[0], shards[1]
    for a, b in [(1, 1), (2, 3), tuple(int(v) for v in rng.integers(1, 256, 2))]:
        mix = rn.MUL[a, c1] ^ rn.MUL[b, c2]
        want = rn.MUL[a, sketch(oracle, c1, seed).view(np.uint8)] ^ rn.MUL[b, sketch(oracle, c2, seed).view(np.uint8)]
        assert (sketch(oracle, mix, seed).view(np.uint8) == want).all()


@pytest.mark.parametrize("k,m", [(3, 2), (6, 3)])
def test_page_oracle_meets_the_guarantee_for_every_damaged_set(oracle, k, m):
    """For every D with |D| <= m and every radius: |D| <= t blames exactly D, t < |D| <= m-t is uncorrectable, and
    anything beyond is flagged.  Damage is random bytes at random places of page 1 of 2."""
    n = PAGE + 700
    shards = clean_set(k, m, n, 99)
    rng = np.random.default_rng(k * 7 + m)
    for size in range(1, m + 1):
        for dset in itertools.combinations(range(k + m), size):
            seed = int(rng.integers(0, 1 << 63))
            bad = [s.copy() for s in shards]
            for i in dset:
                at = rng.choice(np.arange(PAGE, n), size=int(rng.integers(1, 40)), replace=False)
                bad[i][at] ^= rng.integers(1, 256, len(at), dtype=np.uint8)
            sk = [sketch(oracle, s, seed) for s in bad]
            for t in range(0, m // 2 + 1):
                got = page_oracle(sk, k, m, t)
                assert [g for g, _, _ in got] == [1], (dset, t)
                if size <= t:
                    assert got == [(1, mask_of(dset), False)], (dset, t)
                elif size <= m - t:
                    assert got == [(1, 0, True)], (dset, t)


def _locate_raw(L, enc_h, sketches, shard_len, radius, pages, cap, n, per, ok):
    return L.swec_locate_sketch_damage(enc_h, sketches, shard_len, radius, pages, cap, n, per, ok)


def test_argument_rules_before_any_device_work(swec, tmp_path):
    from seaweedfs_b200._native import SketchPage
    ec = swec.erasure_coding
    L = swec.lib()
    enc = ec.Encoder(3, 2, device=-1)
    words = [np.zeros(2, dtype=np.uint64) for _ in range(5)]
    arr = (C.c_void_p * 5)(*[w.ctypes.data for w in words])
    pages, n, per, ok = (SketchPage * 4)(), C.c_int64(0), (C.c_uint64 * 32)(), C.c_int(0)
    args = dict(enc_h=enc._h, sketches=arr, shard_len=PAGE + 1, radius=1, pages=pages, cap=4, n=C.byref(n), per=per,
                ok=C.byref(ok))

    def call(**over):
        return _locate_raw(L, **{**args, **over})
    assert call(enc_h=None) == -1
    assert call(sketches=None) == -1
    assert call(n=None) == -1 and call(ok=None) == -1
    assert call(shard_len=-1) == -1
    assert call(cap=-1) == -1 and call(pages=None) == -1
    assert call(pages=None, cap=0) == -7
    assert call(radius=-1) == -1 and call(radius=3) == -1
    assert call(radius=2) == -1                          # 2·2 > m = 2
    assert call(radius=0) == -7 and call(per=None) == -7
    missing = (C.c_void_p * 5)(*[w.ctypes.data for w in words[:4]], None)
    assert call(sketches=missing) == -2                  # a lost shard: rebuild first
    assert call(sketches=missing, radius=3) == -1        # argument errors first
    assert call() == -7
    with pytest.raises(swec.SwecError) as e:
        enc.locate_sketch_damage(words, [PAGE + 1] * 4 + [PAGE + 2])
    assert e.value.name == "SWEC_ERR_SHARD_SIZE"
    with pytest.raises(swec.SwecError) as e:
        enc.locate_sketch_damage(words[:4] + [None], PAGE + 1)
    assert e.value.name == "SWEC_ERR_TOO_FEW_SHARDS"

    # the device call: argument errors, then the device
    buf = (C.c_uint64 * 4)()
    assert L.swec_page_sketch_device(0, None, 10, 0, 1, buf, None) == -1
    assert L.swec_page_sketch_device(0, buf, 10, 0, 1, None, None) == -1
    assert L.swec_page_sketch_device(0, buf, 10, 100, 1, buf, None) == -1
    assert L.swec_page_sketch_device(0, buf, 10, 0, 1, C.addressof(buf) + 4, None) == -1
    assert L.swec_page_sketch_device(-1, buf, 10, 4096, 1, buf, None) == -7
    assert L.swec_page_sketch_device(-1, None, 0, 0, 1, None, None) == -7

    # the file call: arguments, then the file, then the device; an empty file has no pages and needs no GPU
    ln, npg = C.c_int64(-5), C.c_int64(-5)
    assert L.swec_page_sketch_file(None, 0, 1, buf, 4, C.byref(ln), C.byref(npg)) == -1
    assert L.swec_page_sketch_file(b"x", 0, 1, buf, -1, C.byref(ln), C.byref(npg)) == -1
    assert L.swec_page_sketch_file(b"x", 0, 1, None, 4, C.byref(ln), C.byref(npg)) == -1
    assert L.swec_page_sketch_file(b"x", 0, 1, buf, 4, None, C.byref(npg)) == -1
    assert L.swec_page_sketch_file(str(tmp_path / "nope.ec00").encode(), -1, 1, buf, 4, C.byref(ln), C.byref(npg)) == -4
    empty = tmp_path / "empty.ec00"
    empty.write_bytes(b"")
    assert L.swec_page_sketch_file(str(empty).encode(), -1, 1, None, 0, C.byref(ln), C.byref(npg)) == 0
    assert (ln.value, npg.value) == (0, 0)
    full = tmp_path / "one.ec00"
    full.write_bytes(b"\1" * 5000)
    assert L.swec_page_sketch_file(str(full).encode(), -1, 1, buf, 4, C.byref(ln), C.byref(npg)) == -7


# ---------------------------------------------------------------------------------------------------------- GPU

def _dev_sketch(torch, enc, host: np.ndarray, seed: int, first_column: int = 0, offset: int = 0, stream=None):
    """Device sketches of `host` placed `offset` bytes into a device buffer, on `stream`, with 4 sentinel words after
    the output; returns (sketches, sentinels intact)."""
    n = len(host)
    buf = torch.zeros(n + offset + 16, dtype=torch.uint8, device="cuda")
    if n:
        buf[offset:offset + n] = torch.from_numpy(host).cuda()
    pages = (n + PAGE - 1) // PAGE
    out = torch.full((pages + 4,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device="cuda")
    s = stream or torch.cuda.current_stream()
    torch.cuda.synchronize()
    enc.page_sketch_device(buf.data_ptr() + offset, n, out.data_ptr(), seed, first_column, s.cuda_stream)
    s.synchronize()
    got = out.cpu().numpy().view(np.uint64)
    return got[:pages].copy(), bool((got[pages:] == 0x5A5A5A5A5A5A5A5A).all())


@pytest.mark.gpu
def test_device_sketches_are_the_oracle(swec, cuda, oracle):
    torch = cuda
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    side = torch.cuda.Stream()
    rng = np.random.default_rng(5)
    seeds = [0, MASK64, int(rng.integers(0, 1 << 63)) * 2 + 1]
    firsts = [0, 4096, 1 << 32, 3 * (1 << 30) - 4096]
    lengths = [1, 15, 16, 17, 4095, 4096, 4097, 65 * 4096 + 5, (1 << 20) + 3]
    for n in lengths:
        host = rng.integers(0, 256, n, dtype=np.uint8)
        for i, (seed, first) in enumerate(itertools.product(seeds, firsts)):
            offsets = range(16) if n <= 4097 else (0, 1 + i % 15)
            want = sketch(oracle, host, seed, first)
            for off in offsets:
                got, intact = _dev_sketch(torch, enc, host, seed, first, off, side if off % 2 else None)
                assert intact, (n, seed, first, off)
                assert (got == want).all(), (n, seed, first, off)


@pytest.mark.gpu
def test_pieces_concatenate_across_the_256_mib_piece(swec, cuda, oracle):
    """A shard just over 256 MiB: page-aligned pieces concatenate to the whole, and pages on both sides of the 256 MiB
    mark and at the end match the oracle."""
    torch = cuda
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    L = swec.lib()
    n = (256 << 20) + 3 * PAGE + 5
    buf = torch.empty(n + 3, dtype=torch.uint8, device="cuda")
    assert L.swec_synth_fill_device(0, buf.data_ptr(), 0, (n + 3) // 8 * 8, 0xABCDEF, None) == 0
    seed = 0x0DDBA11
    pages = (n + PAGE - 1) // PAGE
    whole = torch.empty(pages, dtype=torch.int64, device="cuda")
    enc.page_sketch_device(buf.data_ptr(), n, whole.data_ptr(), seed)
    parts = torch.empty(pages, dtype=torch.int64, device="cuda")
    cut = (256 << 20) - 2 * PAGE
    enc.page_sketch_device(buf.data_ptr(), cut, parts.data_ptr(), seed)
    enc.page_sketch_device(buf.data_ptr() + cut, n - cut, parts[cut // PAGE:].data_ptr(), seed, cut)
    torch.cuda.synchronize()
    assert torch.equal(whole, parts)
    got = whole.cpu().numpy().view(np.uint64)
    host = buf[:n].cpu().numpy()
    for g in (0, cut // PAGE - 1, cut // PAGE, (256 << 20) // PAGE - 1, (256 << 20) // PAGE, pages - 2):
        lo = g * PAGE
        want = sketch(oracle, host[lo:lo + 2 * PAGE], seed, lo)
        assert (got[g:g + 2] == want[:2]).all(), g
    # unaligned: the same bytes one byte into the buffer, on the byte path
    buf2 = torch.empty(n + 1, dtype=torch.uint8, device="cuda")
    buf2[1:] = buf[:n]
    out2 = torch.empty(pages, dtype=torch.int64, device="cuda")
    enc.page_sketch_device(buf2.data_ptr() + 1, n, out2.data_ptr(), seed)
    torch.cuda.synchronize()
    assert torch.equal(whole, out2)


@pytest.mark.gpu
@pytest.mark.parametrize("direct", [0, 1])
def test_file_sketches_are_the_device_sketches(swec, cuda, tmp_path, direct):
    torch = cuda
    ec = swec.erasure_coding
    L = swec.lib()
    enc = ec.Encoder(10, 4, device=0)
    rng = np.random.default_rng(direct)
    assert L.swec_set_option(b"file_direct_io", direct) == 0
    try:
        for n in (5, 3 * PAGE + 17, (9 << 20) + 5, (16 << 20) + PAGE + 1):
            host = rng.integers(0, 256, n, dtype=np.uint8)
            path = tmp_path / f"s{n}.ec03"
            path.write_bytes(host.tobytes())
            before = os.stat(path).st_mtime_ns
            seed = int(rng.integers(0, 1 << 63))
            got, length = ec.page_sketch_file(str(path), seed)
            want, _ = _dev_sketch(torch, enc, host, seed)
            assert length == n and (got == want).all(), n
            assert os.stat(path).st_mtime_ns == before and path.read_bytes() == host.tobytes()
            # a short cap: only the first two words are written, the count is the whole
            out = np.full(4, 0x77, dtype=np.uint64)
            ln, npg = C.c_int64(0), C.c_int64(0)
            assert L.swec_page_sketch_file(str(path).encode(), 0, seed, out.ctypes.data, 2, C.byref(ln),
                                           C.byref(npg)) == 0
            assert npg.value == (n + PAGE - 1) // PAGE and ln.value == n
            k = min(2, npg.value)
            assert (out[:k] == want[:k]).all() and (out[k:] == 0x77).all()
        ln, npg = C.c_int64(0), C.c_int64(0)
        assert L.swec_page_sketch_file(str(tmp_path / "gone.ec00").encode(), 0, 1, None, 0, C.byref(ln),
                                       C.byref(npg)) == -4
    finally:
        L.swec_set_option(b"file_direct_io", 0)


def _device_sketches(torch, enc, shards, seed):
    return [_dev_sketch(torch, enc, s, seed)[0] for s in shards]


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", CODES)
def test_clean_sets_flag_nothing(swec, cuda, k, m):
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    n = 5 * PAGE + 77
    sk = _device_sketches(cuda, enc, clean_set(k, m, n, 3), 0xFEED)
    for t in range(0, min(2, m // 2) + 1):
        res = enc.locate_sketch_damage(sk, n, radius=t)
        assert res["ok"] and res["n_flagged"] == 0 and res["pages"] == [] and res["shard_pages"] == {}


def _corpus(k, m, n, rng):
    """name -> [(shard, offsets)] of the damage corpus, on a set of n bytes per shard (n not a page multiple)."""
    last = (n - 1) // PAGE * PAGE
    return {
        "one_byte": [(1, [5000])],
        "whole_pages": [(0, list(range(PAGE, 3 * PAGE)))],
        "page_seam": [(2, [PAGE - 1, PAGE])],
        "partial_last_page": [(k - 1, [n - 1, last])],
        "parity_only": [(k, [100, 2 * PAGE + 9]), (k + m - 1, [3 * PAGE])],
        "two_shards_one_column": [(0, [777]), (k, [777])],
        "two_shards_two_columns_one_page": [(1, [8200]), (2, [9000])],
        "three_shards_one_page": [(0, [300]), (1, [301]), (k + 1, [4000])],
        "scattered": [(int(rng.integers(0, k + m)), [int(x)]) for x in rng.integers(0, n, 12)],
    }


def _damage(shards, spec, rng):
    bad = [s.copy() for s in shards]
    for i, offs in spec:
        offs = np.array(offs)
        bad[i][offs] ^= rng.integers(1, 256, len(offs), dtype=np.uint8)
    return bad


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,radius", [(10, 4, 1), (10, 4, 2), (10, 4, 0), (6, 3, 1), (3, 2, 1), (20, 12, 1)])
def test_locate_equals_the_page_oracle(swec, cuda, oracle, k, m, radius):
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    n = 6 * PAGE + 1234
    shards = clean_set(k, m, n, k + m)
    rng = np.random.default_rng(radius * 31 + k)
    for name, spec in _corpus(k, m, n, rng).items():
        seed = int(rng.integers(0, 1 << 63))
        sk = _device_sketches(cuda, enc, _damage(shards, spec, rng), seed)
        want = page_oracle(sk, k, m, radius)
        res = enc.locate_sketch_damage(sk, [n] * (k + m), radius=radius)
        assert res["pages"] == want, name
        assert res["n_flagged"] == len(want) and res["ok"] == (not want)
        per = {}
        for _, mask, _ in want:
            for i in range(k + m):
                if mask >> i & 1:
                    per[i] = per.get(i, 0) + 1
        assert res["shard_pages"] == per, name
        flagged = {o // PAGE for _, offs in spec for o in offs}
        assert {g for g, _, _ in want} == flagged, name
        if name == "two_shards_two_columns_one_page" and radius == 1:
            assert want == [(2, 0, True)]                 # per page, not per column


def _generate(swec, tmp_path, k, m, seed):
    """A generated RS(k,m) set with each shard file moved into a directory of its own: (base, dirs, files)."""
    ec = swec.erasure_coding
    base_dir = tmp_path / "base"
    base_dir.mkdir()
    base = str(base_dir / "7")
    rng = np.random.default_rng(seed)
    # 9 rows of 10,000-byte blocks: 90,000-byte shards, whose last page is partial
    (base_dir / "7.dat").write_bytes(rng.integers(0, 256, k * 10000 * 8 + 1234, dtype=np.uint8).tobytes())
    ec.generate_ec_files(base, 1000, 1000000, 10000, ec.ECContext(k, m, device=0))
    dirs, files = [], []
    for i in range(k + m):
        d = tmp_path / f"server{i}"
        d.mkdir()
        dst = d / ("7" + ec.ToExt(i))
        os.rename(base + ec.ToExt(i), dst)
        dirs.append(str(d))
        files.append(str(dst))
    return base, dirs, files


def _read_page(path, g, n):
    with open(path, "rb") as f:
        f.seek(g * PAGE)
        return np.frombuffer(f.read(min(PAGE, n - g * PAGE)), dtype=np.uint8).copy()


def _write_page(path, g, data):
    fd = os.open(path, os.O_WRONLY)
    try:
        assert os.pwrite(fd, data.tobytes(), g * PAGE) == len(data)
        os.fdatasync(fd)
    finally:
        os.close(fd)


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", [(10, 4), (6, 3)])
def test_scrub_a_balanced_set_end_to_end(swec, cuda, tmp_path, k, m):
    """Sketch every shard file where it lies, locate from the sketches, fetch only the flagged pages, repair them and
    write them back: the set is clean again, byte for byte the original, and only the blamed files were written."""
    torch = cuda
    ec = swec.erasure_coding
    enc = ec.Encoder(k, m, device=0)
    base, dirs, files = _generate(swec, tmp_path, k, m, k)
    originals = [open(f, "rb").read() for f in files]
    n = len(originals[0])
    rng = np.random.default_rng(m)
    damage = {1: [5000, 5001], k: [3 * PAGE + 7],                          # data page, parity-only page
              2: [8 * PAGE + 10], 3: [8 * PAGE + 2000],                    # two shards, different columns, one page
              0: [n - 1]}                                                  # the partial last page
    for i, offs in damage.items():
        b = np.frombuffer(originals[i], dtype=np.uint8).copy()
        b[offs] ^= rng.integers(1, 256, len(offs), dtype=np.uint8)
        open(files[i], "wb").write(b.tobytes())
    for f in files:
        os.utime(f, ns=(10**18, 10**18))
    assert not ec.locate_ec_damage(base, dirs, ec.ECContext(k, m, device=0))["ok"]

    seed = int(rng.integers(0, 1 << 63))
    sketches, lengths = zip(*(ec.page_sketch_file(f, seed) for f in files))
    moved = sum(s.nbytes for s in sketches)
    res = enc.locate_sketch_damage(list(sketches), list(lengths), radius=1)
    pages = {g for g, _, _ in res["pages"]}
    assert pages == {5000 // PAGE, 3, 8, (n - 1) // PAGE}
    written = set()
    batch, targets = [], []
    for g, mask, bad in res["pages"]:
        if not bad:   # blamed on mask: k pages from outside it rebuild the blamed pages in one batch
            src = [i for i in range(k + m) if not mask >> i & 1][:k]
            item = [None] * (k + m)
            for i in src:
                item[i] = _read_page(files[i], g, n)
                moved += item[i].nbytes
            batch.append(item)
            targets.append((g, mask))
        else:         # uncorrectable at radius 1: every shard's page, corrected column by column on the GPU
            got = [_read_page(files[i], g, n) for i in range(k + m)]
            moved += sum(x.nbytes for x in got)
            dev = [torch.from_numpy(x).cuda() for x in got]
            rep = enc.correct_damage_device([d.data_ptr() for d in dev], len(got[0]), radius=1)
            torch.cuda.synchronize()
            assert rep["uncorrectable_columns"] == 0
            for i, d in enumerate(dev):
                fixed = d.cpu().numpy()
                if not (fixed == got[i]).all():
                    _write_page(files[i], g, fixed)
                    written.add(i)
    if batch:
        enc.reconstruct_batch(batch, data_only=False)
    for item, (g, mask) in zip(batch, targets):
        for i in range(k + m):
            if mask >> i & 1:
                _write_page(files[i], g, item[i])
                written.add(i)
    assert moved <= 8 * len(sketches[0]) * (k + m) + PAGE * (k + m) * len(pages)
    assert written == set(damage)
    assert ec.locate_ec_damage(base, dirs, ec.ECContext(k, m, device=0))["ok"]
    for i, f in enumerate(files):
        assert open(f, "rb").read() == originals[i], i
        assert (os.stat(f).st_mtime_ns == 10**18) == (i not in damage), i


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,radius", [(10, 4, 1), (6, 3, 1), (10, 4, 2)])
def test_flagged_pages_are_the_locate_ranges(swec, cuda, tmp_path, k, m, radius):
    ec = swec.erasure_coding
    enc = ec.Encoder(k, m, device=0)
    base, dirs, files = _generate(swec, tmp_path, k, m, 40 + radius)
    n = os.path.getsize(files[0])
    rng = np.random.default_rng(radius)
    for i in rng.choice(k + m, 3, replace=False):
        b = np.fromfile(files[i], dtype=np.uint8)
        at = rng.integers(0, n, 4)
        b[at] ^= rng.integers(1, 256, 4, dtype=np.uint8)
        b.tofile(files[i])
    loc = ec.locate_ec_damage(base, dirs, ec.ECContext(k, m, device=0), radius=radius)
    want = {g for _, off, ln in loc["ranges"] for g in range(off // PAGE, (off + ln + PAGE - 1) // PAGE)}
    seed = int(rng.integers(0, 1 << 63))
    sketches, lengths = zip(*(ec.page_sketch_file(f, seed) for f in files))
    res = enc.locate_sketch_damage(list(sketches), lengths[0], radius=radius)
    assert {g for g, _, _ in res["pages"]} == want
