"""The device volume calls at every seam of the two-tier striping: swec_encode_volume_device (the call bench.py times, and
the only way into the blocked encode kernels), swec_extract_data_shard_device and swec_write_dat_device.

encodeDatFile (ec_encoder.go:280-321) cuts a .dat into rows of k large blocks, then rows of k small blocks, the last one
zero-padded.  The engine turns that geometry into launches region by region: one blocked launch over a region of whole
16-byte vectors, one flat launch for a single row, one launch per row when a block, the .dat or a parity stream is not
16-byte aligned (or no specialised kernel exists), and the tail row built in scratch.  `volume_plan` restates that plan;
every GPU case is checked against it by the launch counter, and in a child process by the kernel names torch.profiler
records.  Every case compares every parity byte with the oracle's encode of the image, extracts every data shard
(zero padding included) and writes the .dat back from them; every output buffer has 64 sentinel bytes on either side,
and the buffers a call only reads must stay unchanged.

CPU part: StripeGeometry (volume_format.h) compiled for the host against a plain walk of encodeDatFile; the plan
reaches every path over the grid; the argument rules of the three calls on an encoder without a device.
GPU part: the seam grid × eight block pairs × the codes and options that pick different kernels, pointers at several
offsets; and 2D copies whose row pitch (k · large) is more than 2^31 − 1 bytes."""
import ctypes as C
import json
import math
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_kernel_variants import kernel_id, reset_options, set_options  # noqa: E402

INVALID_ARG, NO_DEVICE = -1, -7
GUARD = 64            # sentinel bytes either side of every buffer
SENTINEL = 0xA5
SEED = 0x5EA3EED5F00DCAFE

# (large, small): power-of-two blocks (shift branch of the blocked kernels), 16-byte multiples that are not (division
# branch), a large block that leaves the small rows' parity 8 bytes off alignment, an unaligned small block, the
# reference's ec_test.go blocks, an unaligned large block, equal blocks (no small row ever), the least vector
BLOCKS = [(4096, 512), (4112, 528), (4104, 512), (4096, 520), (10000, 100), (4100, 100), (512, 512), (16, 16)]
REDUCED_BLOCKS = [(4096, 512), (4104, 512), (10000, 100), (16, 16)]

# name: (k, m, options, block pairs).  use_aot 1 is the hand-written RS(10,4) kernel, use_aot 0 the NVRTC one; m > 8
# has no specialised kernel (table kernel per row); jit 0 takes the table kernel per row too
CODES = {
    "rs10x4_aot": (10, 4, {"use_aot": 1}, BLOCKS),
    "rs10x4_nvrtc": (10, 4, {"use_aot": 0}, BLOCKS),
    "rs6x3": (6, 3, {}, BLOCKS),
    "rs1x3": (1, 3, {}, REDUCED_BLOCKS),
    "rs31x1": (31, 1, {}, REDUCED_BLOCKS),
    "rs20x12": (20, 12, {}, REDUCED_BLOCKS),
    "rs6x3_jit0": (6, 3, {"jit": 0}, REDUCED_BLOCKS),
}

# pointer offsets from 16-byte alignment: (label, .dat, parity p at pattern[p % len], extracted shards, write_dat output);
# the grid's cases take them in turn
OFFSETS = [
    ("aligned", 0, (0,), 0, 0),
    ("dat+1", 1, (0,), 0, 0),
    ("dat+8", 8, (0,), 0, 0),
    ("parity 0,+8", 0, (0, 8), 0, 0),
    ("parity +8,0,+4", 0, (8, 0, 4), 0, 0),
    ("shards+3 out+5", 0, (0,), 3, 5),
]


def seam_sizes(k, large, small):
    """.dat sizes at every seam of the striping: the least sizes, around one small row, every tail-block edge, the most
    small rows (R_L - 1), around one and two large rows, and every tail-block edge after 2 large + 3 small rows."""
    rl, rs = k * large, k * small
    s = {0, 1, 15, 16, 17, rs - 1, rs, rs + 1, rl - 1, rl, rl + 1, rl + rs - 1, rl + rs + 1, rl + 3 * rs, 2 * rl - 1,
         2 * rl + 1}
    for j in range(1, k + 1):
        s |= {j * small - 1, j * small + 1}
    for j in range(k + 1):
        s |= {2 * rl + 3 * rs + j * small - 1, 2 * rl + 3 * rs + j * small + 1}
    return sorted(x for x in s if x >= 0)


def grid(name):
    """(large, small, dat_size, offsets) of every case of a code, the offsets taken in turn"""
    k = CODES[name][0]
    cases = [(large, small, n) for large, small in CODES[name][3] for n in seam_sizes(k, large, small)]
    return [c + (OFFSETS[i % len(OFFSETS)],) for i, c in enumerate(cases)]


# ---------------------------------------------------------------- the striping and the launch plan, restated

def stripe_walk(dat_size, k, large, small):
    """encodeDatFile's two loops: rows of (loop, .dat offset, block size, bytes of the .dat in the row)"""
    rows, rem, pos = [], dat_size, 0
    while rem >= k * large:
        rows.append(("large", pos, large, k * large))
        rem, pos = rem - k * large, pos + k * large
    while rem > 0:
        rows.append(("small", pos, small, min(rem, k * small)))
        rem, pos = rem - k * small, pos + k * small
    return rows


def walk_geometry(dat_size, k, large, small):
    """Every field of StripeGeometry, from the walk: the tail is the small row the .dat does not fill, and block i of
    it holds the .dat bytes that fall in [pos + i·small, pos + (i+1)·small)."""
    rows = stripe_walk(dat_size, k, large, small)
    large_rows = [r for r in rows if r[0] == "large"]
    small_full = [r for r in rows if r[0] == "small" and r[3] == k * small]
    tail_row = [r for r in rows if r[0] == "small" and r[3] < k * small]
    assert rows == large_rows + small_full + tail_row and len(tail_row) <= 1
    small_dat = small_full[0][1] if small_full else (tail_row[0][1] if tail_row else dat_size)
    tail_dat = tail_row[0][1] if tail_row else dat_size
    tail = tail_row[0][3] if tail_row else 0
    tail_bytes = [max(0, min(dat_size, tail_dat + (i + 1) * small) - (tail_dat + i * small)) for i in range(k)]
    return {"large_rows": len(large_rows), "small_rows": len(small_full), "tail": tail, "small_dat_offset": small_dat,
            "tail_dat_offset": tail_dat, "small_shard_offset": len(large_rows) * large,
            "tail_shard_offset": len(large_rows) * large + len(small_full) * small,
            "shard_size": sum(r[2] for r in rows), "tail_bytes": tail_bytes}


def specialised(k, m, opts):
    """a Horner kernel exists for the parity rows: the RS(10,4) one compiled with the library, or an NVRTC one"""
    return bool(((k, m) == (10, 4) and opts.get("use_aot", 1)) or (m <= 8 and opts.get("jit", 1)))


def vector_ids(k, m, opts, blocked):
    """The launches of one apply's 16-byte-vector part: the RS(10,4) kernel (enc_threads 512, enc_unroll 2, the boost
    instruction mix: the library's defaults), the NVRTC kernel, or the table kernel per group of at most four rows."""
    if (k, m) == (10, 4) and opts.get("use_aot", 1):
        return [("rs10x4_encode", 512, 2, blocked, False)]
    if m <= 8 and opts.get("jit", 1):
        return [("swec_jit_blocked",) if blocked else ("swec_jit_flat",)]
    assert not blocked
    return [("swec_table_kernel", 10 if k == 10 else 0)] * math.ceil(m / 4)


def volume_plan(k, m, opts, dat_size, large, small, dat_mod, parity_mods):
    """The kernels swec_encode_volume_device launches, in order, for a .dat at address ≡ dat_mod and parity streams at
    addresses ≡ parity_mods (mod 16).  Raises ValueError where the engine would refuse the call."""
    horner = specialised(k, m, opts)

    def apply(in_mods, out_mods, n, blocked, block):
        aligned = all(x % 16 == 0 for x in in_mods + out_mods) and (not blocked or block % 16 == 0)
        nvec = n // 16 if aligned else 0
        tail = n - 16 * nvec
        if blocked and (not aligned or tail):
            raise ValueError("blocked layout needs 16-byte aligned blocks")
        byte_groups = math.ceil(m / 4) if tail else 0
        return (vector_ids(k, m, opts, blocked) if nvec else []) + [("swec_bytes_kernel",)] * byte_groups

    def region(base, block, nrows, poff):
        outs = [p + poff for p in parity_mods]
        vec_ok = horner and block % 16 == 0 and base % 16 == 0 and all(o % 16 == 0 for o in outs)
        if vec_ok or nrows == 1:
            return apply([base + i * block for i in range(k)], outs, nrows * block, nrows > 1, block)
        return [x for r in range(nrows)
                for x in apply([base + (r * k + i) * block for i in range(k)], [o + r * block for o in outs], block,
                               False, block)]

    g = walk_geometry(dat_size, k, large, small)
    plan = []
    if g["large_rows"]:
        plan += region(dat_mod, large, g["large_rows"], 0)
    if g["small_rows"]:
        plan += region(dat_mod + g["small_dat_offset"], small, g["small_rows"], g["small_shard_offset"])
    if g["tail"]:
        plan += region(0, small, 1, g["tail_shard_offset"])      # the zero-padded row, in fresh (aligned) scratch
    return plan


def parity_offsets(m, pattern):
    return [pattern[p % len(pattern)] for p in range(m)]


# ================================================================ CPU part

GEOMETRY_FIELDS = ["large_rows", "small_rows", "tail", "small_dat_offset", "tail_dat_offset", "small_shard_offset",
                   "tail_shard_offset", "shard_size"]


@pytest.fixture(scope="module")
def geometry_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("geometry")
    src = d / "geometry.cc"
    src.write_text('#include "%s"\n' % os.path.join(ROOT, "seaweedfs_b200", "csrc", "volume_format.h") + r'''
extern "C" void geometry(int64_t dat_size, int k, int64_t large, int64_t small, int64_t* out) {
    const swec::StripeGeometry g(dat_size, k, large, small);
    const int64_t v[] = {g.large_rows, g.small_rows, g.tail, g.small_dat_offset(), g.tail_dat_offset(),
                         g.small_shard_offset(), g.tail_shard_offset(), g.shard_size()};
    for (int i = 0; i < 8; i++) out[i] = v[i];
    for (int i = 0; i < k; i++) out[8 + i] = g.tail_bytes(i);
}
''')
    so = str(d / "libgeometry.so")
    subprocess.run(["c++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"), "-o", so,
                    str(src)], check=True)
    L = C.CDLL(so)
    L.geometry.argtypes = [C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_void_p]
    return L


def host_geometry(L, dat_size, k, large, small):
    out = np.zeros(8 + k, dtype=np.int64)
    L.geometry(dat_size, k, large, small, out.ctypes.data)
    g = dict(zip(GEOMETRY_FIELDS, map(int, out[:8])))
    g["tail_bytes"] = [int(x) for x in out[8:]]
    return g


def test_stripe_geometry_is_the_walk_of_encodedatfile(geometry_lib, oracle):
    """StripeGeometry, compiled for the host, field by field against the walk and its shard size against the oracle's:
    every code × block pair × seam size of the GPU grid, and the production blocks at 30 GiB and 30,000 MiB + 123,457
    for k = 1…31."""
    cases = {(CODES[n][0], large, small, size) for n in CODES for large, small, size, _ in grid(n)}
    cases |= {(k, 1 << 30, 1 << 20, size) for k in range(1, 32) for size in (30 << 30, 30000 * (1 << 20) + 123_457)}
    for k, large, small, size in sorted(cases):
        got = host_geometry(geometry_lib, size, k, large, small)
        want = walk_geometry(size, k, large, small)
        assert got == want, (k, large, small, size)
        assert got["shard_size"] == oracle.expected_shard_size(size, k, large, small), (k, large, small, size)


def test_the_grid_reaches_every_path():
    """Over the grid the plan takes every path: blocked and flat vector launches, launches per row, byte launches, the
    tail row; and the regions the engine refused before a parity stream's alignment counted (misaligned parity, or the
    small rows' parity offset off alignment, under a blocked layout) are in it."""
    for name, (k, m, opts, _) in CODES.items():
        ids, refused_before = set(), 0
        for large, small, n, (_, dat_off, pat, _, _) in grid(name):
            pm = parity_offsets(m, pat)
            ids |= set(volume_plan(k, m, opts, n, large, small, dat_off, pm))
            g = walk_geometry(n, k, large, small)
            horner = specialised(k, m, opts)
            for block, rows, base, poff in ((large, g["large_rows"], dat_off, 0),
                                            (small, g["small_rows"], dat_off + g["small_dat_offset"],
                                             g["small_shard_offset"])):
                if horner and rows > 1 and block % 16 == 0 and base % 16 == 0 and any((p + poff) % 16 for p in pm):
                    refused_before += 1
        assert ("swec_bytes_kernel",) in ids, name
        if specialised(k, m, opts):
            assert {x for x in ids if x[0] != "swec_bytes_kernel"} == set(vector_ids(k, m, opts, True) +
                                                                          vector_ids(k, m, opts, False)), (name, ids)
            assert refused_before > 0, name
        else:
            assert ids == {("swec_table_kernel", 10 if k == 10 else 0), ("swec_bytes_kernel",)}, (name, ids)
    # the two shapes of the defect, on RS(10,4): misaligned parity at ec_test.go's blocks with 2 large rows, and the
    # small rows of (4104, 512) whose parity starts 4104 ≡ 8 (mod 16) into each aligned parity buffer
    assert volume_plan(10, 4, {}, 2 * 100_000, 10000, 100, 0, [0, 8, 0, 8]) == [("swec_bytes_kernel",)] * 2
    assert volume_plan(10, 4, {}, 56_400, 4104, 512, 0, [0] * 4) == [("swec_bytes_kernel",)] * 4
    assert volume_plan(10, 4, {}, 2 * 100_000, 10000, 100, 0, [0] * 4) == [("rs10x4_encode", 512, 2, True, False)]


@pytest.mark.parametrize("k,m", [(10, 4), (6, 3), (20, 12), (1, 3), (31, 1)])
def test_argument_rules_before_any_device_work(swec, k, m):
    """On an encoder opened with device -1, every bad argument of the three calls is SWEC_ERR_INVALID_ARG (before the
    device is asked for), and valid arguments reach the device: SWEC_ERR_NO_DEVICE.  NULL entries of the parity and
    data-shard arrays included; no pointer here is ever dereferenced."""
    L = swec.lib()
    enc = swec.erasure_coding.Encoder(k, m, device=-1)
    h = enc._h
    fake = 1 << 24                 # stands for device memory; never touched
    good = dict(dat=fake, size=10 * k * 4096 + 77, large=4096, small=512)

    def arr(n, null=None):
        return (C.c_void_p * n)(*[None if i == null else fake + i * 4096 for i in range(n)])

    def encode(dat=good["dat"], size=good["size"], large=good["large"], small=good["small"], parity="ok"):
        p = arr(m) if parity == "ok" else (None if parity is None else arr(m, null=parity))
        return L.swec_encode_volume_device(h, dat, size, large, small, p, None)

    def extract(dat=good["dat"], size=good["size"], large=good["large"], small=good["small"], sid=0, out=fake):
        return L.swec_extract_data_shard_device(h, dat, size, large, small, sid, out, None)

    def write_dat(shards="ok", size=good["size"], large=good["large"], small=good["small"], out=fake):
        s = arr(k) if shards == "ok" else (None if shards is None else arr(k, null=shards))
        return L.swec_write_dat_device(h, s, size, large, small, out, None)

    try:
        bad = [encode(dat=None), encode(parity=None), encode(size=-1), encode(large=0), encode(large=-1),
               encode(small=0), encode(small=-4096)] + [encode(parity=p) for p in range(m)]
        bad += [extract(dat=None), extract(out=None), extract(sid=-1), extract(sid=k), extract(size=-1),
                extract(large=0), extract(small=-1)]
        bad += [write_dat(shards=None), write_dat(out=None), write_dat(size=-1), write_dat(large=-1),
                write_dat(small=0)] + [write_dat(shards=i) for i in range(k)]
        assert bad == [INVALID_ARG] * len(bad), bad
        assert L.swec_encode_volume_device(None, fake, 16, 4096, 512, arr(m), None) == INVALID_ARG
        ok = [encode(), encode(size=0), extract(), extract(sid=k - 1), write_dat(), write_dat(size=0)]
        assert ok == [NO_DEVICE] * len(ok), ok
    finally:
        enc.close()


# ================================================================ GPU part

def _expected(oracle, k, m, n, large, small):
    dat = oracle.synth(0, n, SEED + n)
    want = oracle.encode_dat_image(dat, k=k, m=m, buffer_size=math.gcd(large, small), large=large, small=small)
    return dat, want


def _guarded(torch, rows, length, extra=16):
    """rows × (guard, room for a 0…15-byte offset, `length`, guard) of sentinel bytes; 16-byte aligned rows"""
    pitch = -(-(2 * GUARD + extra + length) // 16) * 16
    return torch.full((rows, pitch), SENTINEL, dtype=torch.uint8, device="cuda")


def _untouched_outside(row, start, length):
    return bool((row[:start] == SENTINEL).all()) and bool((row[start + length:] == SENTINEL).all())


def run_case(torch, oracle, L, enc, stream, k, m, opts, large, small, n, offsets):
    """Encode, extract every shard and write the .dat back, on `stream`; every byte checked.  Returns the plan."""
    label, dat_off, pat, sh_off, out_off = offsets
    ctx = (k, m, large, small, n, label)
    dat, want = _expected(oracle, k, m, n, large, small)
    shard = len(want[0])
    pofs = parity_offsets(m, pat)
    s = stream.cuda_stream
    with torch.cuda.stream(stream):
        datbuf = _guarded(torch, 1, n)
        if n:
            datbuf[0, GUARD + dat_off:GUARD + dat_off + n] = torch.from_numpy(dat).to("cuda", non_blocking=False)
        dat_before = datbuf.clone()
        par = _guarded(torch, m, shard)
        # the extracted shards are the first k rows of an allocation twice as tall: a copy with a wrong pitch then reads
        # stale sentinel bytes inside it, which the comparison catches, instead of leaving it
        sh = _guarded(torch, 2 * k, shard)
        out = _guarded(torch, 1, n)
        dat_ptr = datbuf.data_ptr() + GUARD + dat_off
        par_ptr = [par[p].data_ptr() + GUARD + pofs[p] for p in range(m)]
        sh_ptr = [sh[i].data_ptr() + GUARD + sh_off for i in range(k)]
        c0 = L.swec_kernel_launches()
        enc.encode_volume_device(dat_ptr, n, par_ptr, s, large, small)
        for i in range(k):
            enc.extract_data_shard_device(dat_ptr, n, i, sh_ptr[i], s, large, small)
        sh_before = sh.clone()
        enc.write_dat_device(sh_ptr, n, out.data_ptr() + GUARD + out_off, s, large, small)
        launches = L.swec_kernel_launches() - c0
        got_par, got_sh, got_out = par.cpu().numpy(), sh.cpu().numpy(), out.cpu().numpy()[0]
        assert torch.equal(datbuf, dat_before), (ctx, "the .dat was written")
        assert torch.equal(sh, sh_before), (ctx, "write_dat wrote to its data shards")
    plan = volume_plan(k, m, opts, n, large, small, dat_ptr % 16, [p % 16 for p in par_ptr])
    for p in range(m):
        start = GUARD + pofs[p]
        assert np.array_equal(got_par[p, start:start + shard], want[k + p]), (ctx, "parity", p)
        assert _untouched_outside(got_par[p], start, shard), (ctx, "parity guard", p)
    for i in range(k):
        start = GUARD + sh_off
        assert np.array_equal(got_sh[i, start:start + shard], want[i]), (ctx, "data shard", i)
        assert _untouched_outside(got_sh[i], start, shard), (ctx, "data shard guard", i)
    assert bool((got_sh[k:] == SENTINEL).all()), (ctx, "written past the shards")
    assert np.array_equal(got_out[GUARD + out_off:GUARD + out_off + n], dat), (ctx, "write_dat")
    assert _untouched_outside(got_out, GUARD + out_off, n), (ctx, "write_dat guard")
    assert launches == len(plan), (ctx, launches, plan)
    return plan


def sweep(torch, oracle, swec, name, stride=1):
    """Every `stride`-th case of a code's grid on a non-default stream, under the code's options; the plans, in order."""
    k, m, opts, _ = CODES[name]
    L = swec.lib()
    reset_options(L)
    set_options(L, **opts)
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    stream = torch.cuda.Stream()
    try:
        return [run_case(torch, oracle, L, enc, stream, k, m, opts, large, small, n, offs)
                for large, small, n, offs in grid(name)[::stride]]
    finally:
        enc.close()
        reset_options(L)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CODES))
def test_volume_calls_at_every_seam(cuda, swec, oracle, name):
    """Every case of the code's grid: parity, extracted shards and the written-back .dat byte for byte, the guards, the
    read-only buffers, and the launch count of the plan."""
    plans = sweep(cuda, oracle, swec, name)
    assert len(plans) == len(grid(name))


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,large,small,n,pattern", [
    (10, 4, 10000, 100, 2 * 10 * 10000, (0, 8)),          # ec_test.go's blocks, 2 large rows, parity 1 and 3 at +8
    (10, 4, 4104, 512, 10 * 4104 + 3 * 10 * 512, (0,)),   # aligned buffers; the small rows' parity starts at 4104 ≡ 8
    (6, 3, 4096, 512, 2 * 6 * 4096 + 17, (3,)),           # every parity stream at +3, through the NVRTC kernels
], ids=["misaligned_parity", "large_block_4104", "rs6x3_parity+3"])
def test_blocked_regions_with_parity_off_alignment(cuda, swec, oracle, k, m, large, small, n, pattern):
    """A region of two or more rows of aligned blocks whose parity streams are not 16-byte aligned takes one launch
    per row instead of being refused (SWEC_ERR_INVALID_ARG, "blocked layout needs 16-byte aligned blocks")."""
    L = swec.lib()
    enc = swec.erasure_coding.Encoder(k, m, device=0)
    try:
        plan = run_case(cuda, oracle, L, enc, cuda.cuda.Stream(), k, m, {}, large, small, n,
                        ("parity " + repr(pattern), 0, pattern, 0, 0))
    finally:
        enc.close()
    assert plan and all(x == ("swec_bytes_kernel",) for x in plan), plan


def _profile_child():
    """In a process of its own (the profiler's CUPTI state stays out of the suite's): every 3rd case of every code under
    torch.profiler; prints RESULT <json>: per code, the plans and the matrix-apply kernels recorded, in launch order."""
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    import seaweedfs_b200 as swec
    from oracle import pyoracle as oracle
    out = {}
    for name in CODES:
        sweep(torch, oracle, swec, name, stride=3)            # NVRTC compiles and table uploads out of the window
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            plans = sweep(torch, oracle, swec, name, stride=3)
            torch.cuda.synchronize()
        events = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA), key=lambda e: e.time_range.start)
        ids = [i for i in map(kernel_id, (e.name for e in events)) if i is not None]
        out[name] = {"plan": [x for p in plans for x in p], "ids": ids if events else None}
    print("RESULT " + json.dumps(out))


@pytest.mark.gpu
def test_kernel_names_are_the_plans(cuda):
    """The kernels torch.profiler records over every 3rd case of every code are exactly the plans', in order; in
    particular an aligned RS(10,4) region of two or more rows still runs the blocked rs10x4_encode instantiation."""
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; import test_volume_device_exhaustive as t; t._profile_child()"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(next(ln for ln in r.stdout.splitlines() if ln.startswith("RESULT "))[7:])
    for name, rec in res.items():
        plan = [tuple(x) for x in rec["plan"]]
        if rec["ids"] is None:
            warnings.warn(f"torch.profiler recorded no kernels (CUPTI unavailable?): kernel names of {name} not checked")
            continue
        assert [tuple(x) for x in rec["ids"]] == plan, name
    assert ("rs10x4_encode", 512, 2, True, False) in {tuple(x) for x in res["rs10x4_aot"]["plan"]}
    assert ("swec_jit_blocked",) in {tuple(x) for x in res["rs10x4_nvrtc"]["plan"]}


# ---------------------------------------------------------------- row pitches above 2^31 - 1

def _cudart():
    # the runtime torch has loaded, found by its soname; else the toolkit's
    for cand in ("libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
        try:
            return C.CDLL(cand)
        except OSError:
            continue
    pytest.skip("no libcudart to ask cudaDevAttrMaxPitch")


def max_pitch():
    v = C.c_int(0)
    assert _cudart().cudaDeviceGetAttribute(C.byref(v), 11, 0) == 0    # cudaDevAttrMaxPitch
    return v.value


def _digest(swec, t, n, s):
    d = C.c_uint64(0)
    assert swec.lib().swec_digest_device(0, t.data_ptr(), n, C.byref(d), s) == 0
    return d.value


PITCH_CASES = [
    # RS(30,2), 72 MiB large blocks: a 2,160 MiB large row; 2 large rows, 3 small rows and a tail (about 9 GiB of HBM)
    (30, 2, 72 << 20, 1 << 20, 2 * 30 * (72 << 20) + 3 * 30 * (1 << 20) + 5 * (1 << 20) + 12_345),
    # the production geometry: a 10 GiB large row; 2 large rows, 1 small row and a tail (about 48 GiB of HBM)
    (10, 4, 1 << 30, 1 << 20, (20 << 30) + (10 << 20) + 12_345),
]


@pytest.mark.gpu
@pytest.mark.parametrize("k,m,large,small,dat_size", PITCH_CASES)
def test_volume_calls_with_row_pitch_above_2_gib(cuda, swec, oracle, k, m, large, small, dat_size):
    """extract and write_dat copy each data shard's blocks out of (into) rows of k·large bytes, more than
    cudaDevAttrMaxPitch allows a 2D copy: every extracted shard and the parity against the CPU oracle's digests of the
    seeded volume, and write_dat gives back the image's device digest.  Measured on an H100 80GB HBM3 (700 W power
    limit): cudaDevAttrMaxPitch is 2,147,483,647, and the runtime still carries out these device-to-device 2D copies
    exactly, so the calls keep one 2D copy per region; this test is what would show a runtime that refuses them."""
    torch, ec = cuda, swec.erasure_coding
    print(f"cudaDevAttrMaxPitch = {max_pitch()}")
    shard = ec.expected_shard_size(dat_size, k, large, small)
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < dat_size + (k + m) * shard + (1 << 30):
        pytest.skip(f"not enough HBM free ({free >> 20} MiB)")
    stream = torch.cuda.Stream()
    s = stream.cuda_stream
    enc = ec.Encoder(k, m, device=0)
    try:
        with torch.cuda.stream(stream):
            dat = torch.empty(dat_size + (-dat_size) % 8, dtype=torch.uint8, device="cuda")
            assert swec.lib().swec_synth_fill_device(0, dat.data_ptr(), 0, dat.numel(), SEED, s) == 0
            dat_digest = _digest(swec, dat, dat_size, s)
            par = [torch.empty(shard, dtype=torch.uint8, device="cuda") for _ in range(m)]
            enc.encode_volume_device(dat.data_ptr(), dat_size, [p.data_ptr() for p in par], s, large, small)
            sh = [torch.empty(shard, dtype=torch.uint8, device="cuda") for _ in range(k)]
            for i in range(k):
                enc.extract_data_shard_device(dat.data_ptr(), dat_size, i, sh[i].data_ptr(), s, large, small)
            got = [_digest(swec, t, shard, s) for t in sh + par]
            del dat
            torch.cuda.empty_cache()
            out = torch.empty(dat_size, dtype=torch.uint8, device="cuda")
            enc.write_dat_device([t.data_ptr() for t in sh], dat_size, out.data_ptr(), s, large, small)
            back = _digest(swec, out, dat_size, s)
        want = oracle.volume_digests(dat_size, SEED, k=k, m=m, large=large, small=small,
                                     kind=1 if oracle.gfni_level() else 2)
        assert got[:k] == want[:k], "extracted data shards"
        assert got[k:] == want[k:], "parity"
        assert back == dat_digest, "write_dat"
    finally:
        enc.close()
