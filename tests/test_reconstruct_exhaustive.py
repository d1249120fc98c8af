"""Plain erasure decoding (`Reconstruct` / `ReconstructData`) at every erasure pattern, to the standard of the exhaustive
damage-decoder tests.  A correct reconstruct gives the original shards back byte for byte, so every GPU result here is
compared with the shards the test started from, not with a restatement of the decode.

CPU part (no GPU):
  * the decode plan (`rs_reconstruct_plan` through `swec_reconstruct_matrix`) at every presence mask of RS(10,4) and of
    every code with k + m <= 8, and at the edge masks of RS(31,1), RS(1,31), RS(20,12) and RS(24,8), against
    `rs_numpy.fused_reconstruct_rows`;
  * the kernel generator (`codegen.cc`) on every decode matrix of RS(10,4), with and without shared power chains, and of
    RS(6,3); every 16th RS(10,4) matrix with `--no-basis`, `--no-cse` and `--search-basis`.  The emitted combiners are
    compiled for the host, ~300 to a translation unit, and checked word by word against the oracle's multiplication
    table.  Every volume rebuild of a pattern that is not compiled in runs an NVRTC kernel built from this text.

GPU part: `swec_reconstruct_device` at every pattern of RS(10,4) on the table kernel, the compiled-in kernels, the NVRTC
kernels and the byte kernel (the path asserted through `swec_jit_stats`); every pattern of the small codes and the edge
masks of the wide ones; one `swec_reconstruct_batch` holding every (pattern, data_only) key of RS(10,4); degraded
needle reads of a mounted volume at every loss pattern of RS(10,4) and RS(6,3)."""
import contextlib
import ctypes as C
import itertools
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_codegen as tcg  # noqa: E402
import test_kernel_variants as tkv  # noqa: E402
import test_volume_ops as tvo  # noqa: E402
from oracle import rs_numpy as rn  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "seaweedfs_b200", "csrc")
SENTINEL = 0xA5
GUARD = 64                                   # bytes either side of every shard on the device, 16-byte aligned
N_DEVICE = 3 * 65536 + 13                    # vectors over several tiles and a 13-byte tail for the byte kernel
PACKED_LIMIT = 2 << 20                       # host_seam.cc packed_max_bytes(): bigger batch items stream
SMALL_CODES = [(k, m) for k in range(1, 8) for m in range(1, 8) if k + m <= 8]


# ================================================================ fixtures

@pytest.fixture
def options(swec):
    """The library's options, back to the documented defaults afterwards (there is no getter)."""
    L = swec.lib()
    tkv.reset_options(L)
    try:
        yield L
    finally:
        tkv.reset_options(L)
        tkv.set_options(L, host_zero_copy=2)


@pytest.fixture(scope="module")
def tool(tmp_path_factory):
    """The generator's command-line front end (codegen_main.cc), built for the host."""
    d = tmp_path_factory.mktemp("codegen")
    exe = str(d / "swec_codegen")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe] + [os.path.join(CSRC, f) for f in
                   ("codegen_main.cc", "codegen.cc", "gf256.cc")], check=True)
    return d, exe


# ================================================================ the oracle's decode plans

@contextlib.contextmanager
def memoised_oracle():
    """rs_numpy.fused_reconstruct_rows with its generator matrices and inverses memoised: the same statement, fast
    enough to be asked for every mask of a code."""
    build, inv = rn.build_matrix, rn.mat_inv
    gens, invs = {}, {}

    def build_matrix(k, total):
        if (k, total) not in gens:
            gens[(k, total)] = build(k, total)
        return gens[(k, total)].copy()

    def mat_inv(m):
        key = (m.shape, m.tobytes())
        if key not in invs:
            invs[key] = inv(m)
        return invs[key].copy()

    rn.build_matrix, rn.mat_inv = build_matrix, mat_inv
    try:
        yield rn.fused_reconstruct_rows
    finally:
        rn.build_matrix, rn.mat_inv = build, inv


def loss_patterns(total, most):
    """Every set of 1..most lost shard ids, by size, then lexicographically."""
    return [c for r in range(1, most + 1) for c in itertools.combinations(range(total), r)]


def decode_matrices(k, m):
    """(lost, data_only, rows) of every pattern of 1..m lost shards with something to rebuild."""
    out = []
    with memoised_oracle() as fused:
        for lost in loss_patterns(k + m, m):
            present = [i not in lost for i in range(k + m)]
            for data_only in (False, True):
                _, outs, rows = fused(k, m, present, data_only)
                if outs:
                    out.append((lost, data_only, rows))
    return out


def edge_masks(k, m, seed=0):
    """The masks item 1 names for the wide codes: RS(31,1) every single loss and none; RS(1,31) every first present
    shard with the rest all present or all missing; RS(20,12) / RS(24,8) seeded masks of every loss count, plus all data
    lost, exactly k present and 8, 9 and 12 lost shards (more than SWEC_MAX_OUTPUTS = 8 outputs, which the table path
    splits into groups of 4 rows)."""
    n = k + m
    if (k, m) == (31, 1):
        return [tuple(i != j for i in range(n)) for j in range(n)] + [(True,) * n]
    if (k, m) == (1, 31):
        return [tuple(i == f or (i > f and rest) for i in range(n)) for f in range(n) for rest in (True, False)]
    rng = np.random.default_rng(seed + 1000 * k + m)
    masks = [tuple(i >= k for i in range(n)), tuple(i >= m for i in range(n)), tuple(i < k for i in range(n))]
    for lost in (8, 9, 12, m, m + 1):
        for _ in range(20):
            gone = set(rng.choice(n, lost, replace=False).tolist())
            masks.append(tuple(i not in gone for i in range(n)))
    for _ in range(300):
        gone = set(rng.choice(n, int(rng.integers(0, m + 3)), replace=False).tolist())
        masks.append(tuple(i not in gone for i in range(n)))
    return masks


# ================================================================ CPU part

def _check_plans(swec, k, m, masks):
    ec = swec.erasure_coding
    enc = ec.Encoder(k, m, device=-1)
    refused = 0
    try:
        with memoised_oracle() as fused:
            for present in masks:
                for data_only in (False, True):
                    if sum(present) < k:
                        with pytest.raises(swec.SwecError) as e:
                            enc.reconstruct_matrix(present, data_only)
                        assert e.value.name == "SWEC_ERR_TOO_FEW_SHARDS", (k, m, present)
                        refused += 1
                        continue
                    valid, missing, rows = fused(k, m, list(present), data_only)
                    ins, outs, got = enc.reconstruct_matrix(present, data_only)
                    assert ins == valid and outs == missing, (k, m, present, data_only, ins, outs)
                    assert got.shape == rows.shape and (got == rows).all(), (k, m, present, data_only)
    finally:
        enc.close()
    return refused


def test_decode_plan_every_mask(swec):
    """swec_reconstruct_matrix against rs_numpy.fused_reconstruct_rows (inputs, outputs and rows) at all 2^14 masks of
    RS(10,4) and all masks of every code with k + m <= 8, data_only 0 and 1; fewer than k present is
    SWEC_ERR_TOO_FEW_SHARDS, exactly then."""
    for k, m in [(10, 4)] + SMALL_CODES:
        masks = list(itertools.product((False, True), repeat=k + m))
        refused = _check_plans(swec, k, m, masks)
        assert refused == 2 * sum(1 for p in masks if sum(p) < k)


@pytest.mark.parametrize("k,m", [(31, 1), (1, 31), (20, 12), (24, 8)])
def test_decode_plan_wide_codes(swec, k, m):
    """The same at the edges of the wide codes: a single parity shard, a single data shard (every first present shard),
    and RS(20,12) / RS(24,8) with all data lost, exactly k present, and 8, 9 and 12 outputs."""
    masks = edge_masks(k, m)
    _check_plans(swec, k, m, masks)
    if m >= 8:
        outs = {sum(1 for p in mask if not p) for mask in masks if sum(mask) >= k}
        assert {8, m} <= outs and (m < 9 or 9 in outs), outs


GEN_HARNESS_MAIN = r"""
template <class G> static void run(unsigned long long s) {
  u32 x[G::K], y[G::R];
  for (int it = 0; it < ITERS; it++) {
    for (int i = 0; i < G::K; i++) { s ^= s << 13; s ^= s >> 7; s ^= s << 17; x[i] = (u32)(s >> 16); }
    if (it == 0) for (int i = 0; i < G::K; i++) x[i] = 0xffffffffu;
    if (it == 1) for (int i = 0; i < G::K; i++) x[i] = 0x80018001u << (i & 3);
    if (it == 2) for (int i = 0; i < G::K; i++) x[i] = 0x80018001u << i;
    G::combine(x, y);
    fwrite(x, 4, G::K, stdout); fwrite(y, 4, G::R, stdout);
  }
}
int main() {
RUNS
  return 0;
}
"""
GEN_ITERS = 48
UNIT = 300


def _emit(exe, name, rows, extra):
    r, k = rows.shape
    return subprocess.run([exe, "--name", name, *extra, "--rows", str(r), str(k)] + [str(int(v)) for v in rows.ravel()],
                          check=True, stdout=subprocess.PIPE, text=True).stdout


def _run_unit(d, idx, cases, texts):
    prelude = tcg.HARNESS.split('#include "gen.inc"')[0]
    runs = "\n".join(f"  run<G{j}>({0x9E3779B97F4A7C15 + j}ull);" for j, _ in cases)
    src = prelude + f"#define ITERS {GEN_ITERS}\n" + "".join(texts[j] for j, _ in cases) + \
        GEN_HARNESS_MAIN.replace("RUNS", runs)
    cc, exe = d / f"unit{idx}.cc", d / f"unit{idx}"
    cc.write_text(src)
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", str(exe), str(cc)], check=True)
    return subprocess.run([str(exe)], check=True, stdout=subprocess.PIPE).stdout


def test_generator_every_decode_matrix(tool):
    """codegen.cc on all 2,925 decode matrices of RS(10,4) (every pattern of 1-4 lost shards, data_only 0 and 1, minus
    the 15 parity-only patterns of ReconstructData, which have no outputs), once with the default options and once with
    --share-powers (both ship: the NVRTC key carries jit_share_powers); all 251 of RS(6,3); every 16th RS(10,4) matrix
    with --no-basis, --no-cse and --search-basis.  Each combiner, under a name of its own, runs on seeded random words,
    all-0xFF words and 0x80018001 shifted per input, and every output word equals the matrix product by rs_numpy.MUL."""
    d, exe = tool
    t0 = time.perf_counter()
    rs10 = decode_matrices(10, 4)
    rs6 = decode_matrices(6, 3)
    assert len(rs10) == 2925 and len({(r.shape, r.tobytes()) for _, _, r in rs10}) == 2085
    assert len(rs6) == 251
    cases = [(rows, ()) for _, _, rows in rs10] + [(rows, ("--share-powers",)) for _, _, rows in rs10]
    cases += [(rows, ()) for _, _, rows in rs6]
    cases += [(rows, (flag,)) for _, _, rows in rs10[::16] for flag in ("--no-basis", "--no-cse", "--search-basis")]
    workers = os.cpu_count() or 4
    with ThreadPoolExecutor(workers) as pool:
        texts = list(pool.map(lambda jc: _emit(exe, f"G{jc[0]}", jc[1][0], jc[1][1]), enumerate(cases)))
        units = [list(enumerate(cases))[i:i + UNIT] for i in range(0, len(cases), UNIT)]
        outs = list(pool.map(lambda iu: _run_unit(d, iu[0], iu[1], texts), enumerate(units)))
    checked = 0
    for unit, raw in zip(units, outs):
        words = np.frombuffer(raw, dtype="<u4")
        pos = 0
        for j, (rows, extra) in unit:
            r, k = rows.shape
            blk = words[pos:pos + GEN_ITERS * (k + r)].reshape(GEN_ITERS, k + r)
            pos += GEN_ITERS * (k + r)
            x = blk[:, :k].copy().view(np.uint8).reshape(-1, k, 4)
            y = blk[:, k:].copy().view(np.uint8).reshape(-1, r, 4)
            want = np.zeros((r, GEN_ITERS, 4), dtype=np.uint8)
            for i in range(k):
                want ^= rn.MUL[rows[:, i]][:, x[:, i, :]]
            bad = np.nonzero((want.transpose(1, 0, 2) != y).any(axis=(0, 2)))[0]
            assert not len(bad), (j, extra, rows.tolist(), "rows", bad.tolist())
            checked += 1
        assert pos == len(words)
    assert checked == len(cases)
    print(f"{checked} combiners checked in {time.perf_counter() - t0:.1f} s on {workers} CPUs")


# ================================================================ GPU part: device buffers

def _stats(L):
    c, h, a = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    L.swec_jit_stats(C.byref(c), C.byref(h), None, C.byref(a))
    return c.value + h.value, a.value


def _pitch(n):
    return tkv.round_up(n + 2 * GUARD, 256)


class DeviceShards:
    """k+m shards of n bytes on the device, each at GUARD bytes into a row of SENTINEL, and the reconstruct of a pattern
    on a copy of them, checked against the originals."""

    def __init__(self, torch, k, m, n, seed):
        self.torch, self.k, self.m, self.n = torch, k, m, n
        rng = np.random.default_rng(seed)
        data = [rng.integers(0, 256, n, dtype=np.uint8) for _ in range(k)]
        full = np.full((k + m, _pitch(n)), SENTINEL, dtype=np.uint8)
        full[:, GUARD:GUARD + n] = np.stack(data + rn.encode(k, m, data))
        self.full = torch.from_numpy(full).cuda()

    def run(self, enc, present, data_only, shift=None):
        """Reconstruct with the missing rows set to SENTINEL; shift = a shard id moves that shard's bytes (and its
        pointer) one byte further into its row.  Returns True iff every byte of every row is as it must be."""
        torch, n, total = self.torch, self.n, self.k + self.m
        full = self.full
        if shift is not None:
            full = full.clone()
            j = shift
            full[j, GUARD + 1:GUARD + 1 + n] = self.full[j, GUARD:GUARD + n].clone()
            full[j, GUARD] = SENTINEL
        start = [GUARD + (1 if i == shift else 0) for i in range(total)]
        work = full.clone()
        lost = [i for i in range(total) if not present[i]]
        for i in lost:
            work[i, start[i]:start[i] + n] = SENTINEL
        ptrs = [work.data_ptr() + i * work.shape[1] + start[i] for i in range(total)]
        enc.reconstruct_device(ptrs, [int(p) for p in present], n, data_only, torch.cuda.current_stream().cuda_stream)
        want = full
        kept = [i for i in lost if i >= self.k] if data_only and sum(present) < total else []
        if kept:                                   # ReconstructData leaves a missing parity shard's buffer alone
            want = full.clone()
            for i in kept:
                want[i, start[i]:start[i] + n] = SENTINEL
        return torch.equal(work, want)


@pytest.fixture(scope="module")
def rs10_device(cuda):
    return DeviceShards(cuda, 10, 4, N_DEVICE, 0x2EC0)


def _rs10_cases():
    """(lost, data_only, rows) of every RS(10,4) pattern, data_only 0 and 1 (2,940 calls, 2,925 with outputs)."""
    with memoised_oracle() as fused:
        return [(lost, d, fused(10, 4, [i not in lost for i in range(14)], d)[2])
                for lost in loss_patterns(14, 4) for d in (False, True)]


def _compiled_in():
    with memoised_oracle() as fused:
        return [fused(10, 4, [i not in lost for i in range(14)])[2] for lost in tkv.RECON_PATTERNS]


@pytest.mark.gpu
def test_device_table_kernel_every_pattern(cuda, swec, options, rs10_device):
    """jit = 0, use_aot = 0: all 2,940 (pattern, data_only) calls of RS(10,4), three times each, on the table kernel
    (and the byte kernel for the tail).  No compiled-in launch and no NVRTC compile or disk hit."""
    L = options
    tkv.set_options(L, jit=0, use_aot=0)
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    cases = _rs10_cases()
    assert sum(1 for _, _, rows in cases if len(rows)) == 2925
    before = _stats(L)
    try:
        for rep in range(3):
            for lost, data_only, _ in cases:
                assert rs10_device.run(enc, [i not in lost for i in range(14)], data_only), (rep, lost, data_only)
    finally:
        enc.close()
    assert _stats(L) == before


@pytest.mark.gpu
def test_device_compiled_in_kernels_every_pattern(cuda, swec, options, rs10_device):
    """Defaults with jit = 0: a call takes a compiled-in reconstruct kernel exactly when its fused matrix equals one of
    the 15 compiled into the library (every single loss and shards 0-3 lost, data_only 0 — and the data_only = 1
    patterns whose matrix is the same, e.g. shard 0 and shard 13 lost), and the table kernel otherwise."""
    L = options
    tkv.set_options(L, jit=0)
    aot = _compiled_in()
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    hits = 0
    try:
        for rep in range(3):
            for lost, data_only, rows in _rs10_cases():
                is_aot = any(rows.shape == a.shape and (rows == a).all() for a in aot)
                c0, a0 = _stats(L)
                assert rs10_device.run(enc, [i not in lost for i in range(14)], data_only), (rep, lost, data_only)
                c1, a1 = _stats(L)
                assert (c1 - c0, a1 - a0) == (0, int(is_aot)), (lost, data_only, is_aot, a1 - a0)
                hits += is_aot
    finally:
        enc.close()
    assert hits > 3 * len(aot), hits        # the data_only twins of the compiled-in matrices take them too


# the NVRTC set, sized by the cold compile time (test_device_nvrtc_kernels): every 1-loss pattern, every 3rd 2-loss
# pattern and every 64th 3- and 4-loss pattern
NVRTC_STRIDES = {1: 1, 2: 3, 3: 64, 4: 64}


def nvrtc_patterns():
    pick = {r: list(itertools.combinations(range(14), r))[::NVRTC_STRIDES[r]] for r in NVRTC_STRIDES}
    one_two = [(lost, False) for r in (1, 2) for lost in pick[r]]
    three_four = pick[3] + pick[4]
    return one_two + [(lost, d) for lost in three_four for d in (False, True)]


def _nvrtc_child():
    """In a fresh process, so that every matrix is new to the in-process kernel cache and costs exactly one NVRTC
    compile or one disk-cache hit.  Prints RESULT <json>."""
    import torch
    import seaweedfs_b200
    from seaweedfs_b200 import erasure_coding as ec
    L = seaweedfs_b200.lib()
    tkv.reset_options(L)
    tkv.set_options(L, jit=1, jit_min_bytes=0, use_aot=0)
    shards = DeviceShards(torch, 10, 4, N_DEVICE, 0x2EC0)
    enc = ec.Encoder(10, 4, device=0)
    bad, distinct, costs = [], set(), []
    t0 = time.perf_counter()
    with memoised_oracle() as fused:
        for rep in range(3):
            for lost, data_only in nvrtc_patterns():
                rows = fused(10, 4, [i not in lost for i in range(14)], data_only)[2]
                c0, a0 = _stats(L)
                if not shards.run(enc, [i not in lost for i in range(14)], data_only):
                    bad.append([list(lost), data_only, rep])
                c1, a1 = _stats(L)
                key = (rows.shape, rows.tobytes())
                costs.append([list(lost), data_only, rep, c1 - c0, a1 - a0, key not in distinct and len(rows) > 0])
                if len(rows):
                    distinct.add(key)
    enc.close()
    print("RESULT " + json.dumps({"bad": bad, "distinct": len(distinct), "costs": costs,
                                  "seconds": time.perf_counter() - t0}))


@pytest.mark.gpu
def test_device_nvrtc_kernels(cuda):
    """jit = 1, jit_min_bytes = 0 (inline compile), use_aot = 0, in a process of its own: every 1-loss and every 3rd
    2-loss pattern with data_only 0, and every 64th 3- and 4-loss pattern with data_only 0 and 1, three times each.  The
    first call of each distinct matrix costs exactly one compile or disk hit, every other call none, and no compiled-in
    kernel runs.  On a cold cubin cache, 151 distinct matrices took 97.5 s on an H100 80GB HBM3 host (700 W power limit):
    0.65 s per matrix, almost all of it NVRTC on the CPU (swec_debug_jit_compile: 0.25 s for one output row, 0.47 s for
    three on a build machine).  This set has ~80 distinct matrices, about 50 s cold."""
    env = dict(os.environ)
    env.pop("SWEC_NO_JIT", None)
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; import test_reconstruct_exhaustive as t; t._nvrtc_child()"
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(next(ln for ln in r.stdout.splitlines() if ln.startswith("RESULT "))[7:])
    assert not res["bad"], res["bad"][:5]
    wrong = [c for c in res["costs"] if c[3] != int(c[5]) or c[4] != 0]
    assert not wrong, wrong[:5]
    assert sum(c[3] for c in res["costs"]) == res["distinct"] > 60
    print(f"{res['distinct']} NVRTC matrices, {res['seconds']:.1f} s")


@pytest.mark.gpu
def test_device_offset_pointer(cuda, swec, options, rs10_device):
    """jit = 0: one pointer of the shards a call reads or writes one byte past 16-byte alignment (a different one per
    call, over a stride of the patterns and the 15 compiled-in ones).  Every byte is right, and the call leaves the
    16-byte vector kernels alone: not even a compiled-in pattern launches its kernel, and nothing is compiled."""
    L = options
    tkv.set_options(L, jit=0)
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    cases = [(lost, d) for lost in tkv.RECON_PATTERNS for d in (False, True)]
    cases += [(lost, d) for j, lost in enumerate(loss_patterns(14, 4)) if j % 23 == 0 for d in (False, True)]
    before = _stats(L)
    try:
        for j, (lost, data_only) in enumerate(cases):
            with memoised_oracle() as fused:
                ins, outs, _ = fused(10, 4, [i not in lost for i in range(14)], data_only)
            if not outs:
                continue
            shift = (ins + outs)[j % (len(ins) + len(outs))]      # a shard the call reads or writes
            assert rs10_device.run(enc, [i not in lost for i in range(14)], data_only, shift=shift), (lost, data_only, shift)
    finally:
        enc.close()
    assert _stats(L) == before


@pytest.mark.gpu
def test_device_small_and_wide_codes(cuda, swec, options):
    """Default options: every pattern of every code with k + m <= 8, and the edge masks of RS(31,1), RS(1,31),
    RS(20,12) and RS(24,8) (test_decode_plan_wide_codes), data_only 0 and 1."""
    ec = swec.erasure_coding
    n = 65536 + 13
    for k, m in SMALL_CODES + [(31, 1), (1, 31), (20, 12), (24, 8)]:
        shards = DeviceShards(cuda, k, m, n, 0x5A11 + 64 * k + m)
        masks = ([tuple(i not in lost for i in range(k + m)) for lost in loss_patterns(k + m, m)]
                 if (k, m) in SMALL_CODES else [p for p in edge_masks(k, m) if sum(p) >= k])
        enc = ec.Encoder(k, m, device=0)
        try:
            for present in masks:
                for data_only in (False, True):
                    assert shards.run(enc, present, data_only), (k, m, present, data_only)
        finally:
            enc.close()


# ================================================================ GPU part: one batch of every key

BATCH_LENGTHS = (1, 15, 16, 17, 4095, 4097, 65539)


def _batch(seed=0xBA7C):
    """Every (pattern, data_only) key of RS(10,4), three items per key with lengths cycling through BATCH_LENGTHS, and
    every 1000th item PACKED_LIMIT + 1 bytes long.  The present shards are slices of one encoded source at per-item
    offsets; each missing shard gets a buffer of its own between two guards in one arena."""
    rng = np.random.default_rng(seed)
    S = 2 * PACKED_LIMIT + 4096
    data = [rng.integers(0, 256, S, dtype=np.uint8) for _ in range(10)]
    src = np.stack(data + rn.encode(10, 4, data))
    items, pos, j = [], 0, 0
    for lost in loss_patterns(14, 4):
        for data_only in (False, True):
            for _ in range(3):
                n = PACKED_LIMIT + 1 if j % 1000 == 500 else BATCH_LENGTHS[j % len(BATCH_LENGTHS)]
                off = int(rng.integers(0, S - n))
                outs = {}
                for i in lost:
                    outs[i] = pos + GUARD
                    pos += n + 2 * GUARD
                items.append((lost, data_only, n, off, outs))
                j += 1
    return src, items, pos


@pytest.mark.gpu
@pytest.mark.parametrize("zero_copy", [0, 1, 2])
def test_reconstruct_batch_every_key(cuda, swec, options, zero_copy):
    """One swec_reconstruct_batch of ~8,800 items on pageable buffers: one group per (pattern, data_only) key, each
    packing its items into a staging slot, the ring turning over thousands of times; a handful of items over the
    packed limit stream through swec_reconstruct.  jit = 0 keeps the ~2,000 cold matrices on the table and
    compiled-in kernels.  Every missing data shard (and parity shard, data_only 0) equals the original; a missing parity
    shard of a data_only item keeps its sentinel; present shards and every guard are untouched.  The call's launches
    stay within one per group plus the streamed items' pieces: it did not fall apart into one call per item."""
    from seaweedfs_b200._native import ReconstructItem
    L = options
    tkv.set_options(L, jit=0, host_zero_copy=zero_copy)
    src, items, arena_len = _batch()
    src_copy = src.copy()
    arena = np.full(arena_len, SENTINEL, dtype=np.uint8)
    want = arena.copy()
    arr = (ReconstructItem * len(items))()
    keep = []
    groups, streamed = set(), 0
    for it, (lost, data_only, n, off, outs) in zip(arr, items):
        ptrs = (C.c_void_p * 14)()
        for i in range(14):
            ptrs[i] = arena.ctypes.data + outs[i] if i in outs else src[i].ctypes.data + off
        present = np.array([i not in lost for i in range(14)], dtype=np.uint8)
        keep.append((ptrs, present))
        it.shards = C.cast(ptrs, C.POINTER(C.c_void_p))
        it.present = present.ctypes.data_as(C.POINTER(C.c_uint8))
        it.shard_len, it.data_only = n, int(data_only)
        for i, p in outs.items():
            if i < 10 or not data_only:
                want[p:p + n] = src[i, off:off + n]
        if (n + 15) & ~15 > PACKED_LIMIT:
            streamed += 1
        elif any(i < 10 or not data_only for i in lost):
            groups.add((lost, data_only))
    assert len(items) == 3 * 2940 and 5 <= streamed <= 10
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    try:
        before = L.swec_kernel_launches()
        swec.erasure_coding.check(L.swec_reconstruct_batch(enc._h, arr, len(items)))
        launches = L.swec_kernel_launches() - before
    finally:
        enc.close()
    assert (src == src_copy).all(), "a present shard was written"
    if not np.array_equal(arena, want):
        first = int(np.argmax(arena != want))
        culprit = next(x for x in items if any(p - GUARD <= first < p + x[2] + GUARD for p in x[4].values()))
        pytest.fail(f"item {culprit[:4]} differs at arena byte {first}")
    # every group's items fit one slot (3 items of at most 65,552 padded bytes); a streamed item is cut into pieces of at
    # least host_min_chunk (256 KiB), each one vector launch plus at most one tail launch
    per_streamed = 2 * -(-(PACKED_LIMIT + 1) // (256 << 10))
    assert len(groups) <= launches <= len(groups) + streamed * per_streamed, (launches, len(groups), streamed)


# ================================================================ GPU part: degraded needle reads

def _record_chunks(dat, live, shard_dat_size, k):
    """(offset, size, expected bytes, [(shard, shard offset, length)] of the read) of every live record."""
    out = []
    for key, off, size in live:
        want = tvo.expected_record(dat, off * 8, size)
        chunks = []
        for iv in rn.locate_data(1 << 30, 1 << 20, shard_dat_size, off * 8, len(want), k):
            sid, soff = rn.interval_to_shard(iv, 1 << 30, 1 << 20, k)
            chunks.append((sid, soff, iv[2]))
        out.append((key, want, chunks))
    return out


# every pattern of m lost shards of RS(6,3); every 8th of RS(10,4)'s 1,001 four-shard losses — a mount and read of all
# 1,470 RS(10,4) patterns took 210 s on an H100 80GB HBM3 host (0.14 s per pattern, most of it creating the volume's
# encoder and staging ring on its first recovery), the 595 kept here about 85 s
FULL_LOSS_STRIDE = {10: 8, 6: 1}


def _ratio_volume(oracle, tmp_path, k, m, seed):
    dat, idx = tvo.synthetic_volume(seed=seed, needles=600)
    base, _ = tvo.lay_down_ec_volume(oracle, tmp_path, dat, idx, k=k, m=m)
    json.dump({"version": 3, "datFileSize": str(len(dat)), "ecShardConfig": {"dataShards": k, "parityShards": m}},
              open(base + ".vif", "w"))
    live = [(key, o, s) for key, o, s in rn._entries(rn.sorted_ecx_from_idx(idx))]
    return base, dat, live


def _read_with(ec, base, away, lost, live):
    """Mount the volume with the shard files in `lost` moved away, read every live record, unmount, put the files
    back."""
    moved = []
    for i in lost:
        os.rename(base + ec.ToExt(i), os.path.join(away, ec.ToExt(i)))
        moved.append(i)
    try:
        vol = ec.EcVolume(base)
        try:
            return vol.read_needles([key for key, _, _ in live])
        finally:
            vol.close()
    finally:
        for i in moved:
            os.rename(os.path.join(away, ec.ToExt(i)), base + ec.ToExt(i))


@pytest.mark.gpu
@pytest.mark.parametrize("k,m", [(10, 4), (6, 3)])
def test_degraded_needle_reads_every_loss_pattern(cuda, swec, oracle, options, tmp_path, k, m):
    """A mounted volume of ~600 records over two small rows (RS(10,4), and RS(6,3) through its .vif): with the shard
    files of each pattern of 1..m lost shards moved away (RS(6,3): all 129; RS(10,4): all 469 of 1-3 lost shards and
    every 8th of the 1,001 four-shard losses, FULL_LOSS_STRIDE), every live record reads back as
    expected_record, with recovered_intervals = the number of its located chunks on lost data shards.  Every 50th
    pattern of m + 1 lost shards: exactly the records with a chunk on a lost data shard are SWEC_ERR_TOO_FEW_SHARDS, the
    others still read, with nothing recovered."""
    ec = swec.erasure_coding
    base, dat, live = _ratio_volume(oracle, tmp_path, k, m, seed=61 + k)
    away = str(tmp_path / "away")
    os.mkdir(away)
    vol = ec.EcVolume(base, device=-1)
    sds = vol.info()["shard_dat_size"]
    vol.close()
    assert sds == len(dat) // k
    recs = _record_chunks(dat, live, sds, k)
    assert len(recs) > 200 and sum(len(c) > 1 for _, _, c in recs) > 0
    t0 = time.perf_counter()
    patterns = loss_patterns(k + m, m - 1) + list(itertools.combinations(range(k + m), m))[::FULL_LOSS_STRIDE[k]]
    assert len(patterns) == {10: 469 + 126, 6: 129}[k]
    for lost in patterns:
        out = _read_with(ec, base, away, lost, live)
        lost_data = {i for i in lost if i < k}
        for r, (key, want, chunks) in zip(out, recs):
            n_lost = sum(1 for c in chunks if c[0] in lost_data)
            assert r["status"] == "SWEC_OK", (lost, key, r["status"])
            assert r["n_bytes"] == len(want) and (r["bytes"] == want).all(), (lost, key)
            assert r["recovered_intervals"] == n_lost, (lost, key, r["recovered_intervals"], n_lost)
    for lost in list(itertools.combinations(range(k + m), m + 1))[::50]:
        out = _read_with(ec, base, away, lost, live)
        lost_data = {i for i in lost if i < k}
        for r, (key, want, chunks) in zip(out, recs):
            if any(c[0] in lost_data for c in chunks):
                assert r["status"] == "SWEC_ERR_TOO_FEW_SHARDS", (lost, key, r["status"])
            else:
                assert r["status"] == "SWEC_OK" and r["recovered_intervals"] == 0, (lost, key, r["status"])
                assert (r["bytes"] == want).all(), (lost, key)
    print(f"RS({k},{m}): {len(patterns)} patterns in {time.perf_counter() - t0:.1f} s")


@pytest.mark.gpu
def test_degraded_needle_reads_with_a_short_shard(cuda, swec, oracle, options, tmp_path):
    """Shard 0 lost and shard 5 cut to half its size: intervals in the first half of the shards are rebuilt from a mask
    without shard 0, those past it from one without 0 and 5, so one call's batch holds several groups.  Every record
    reads back; recovered_intervals counts the chunks on shard 0 and the chunks on shard 5 that reach past the cut."""
    ec = swec.erasure_coding
    base, dat, live = _ratio_volume(oracle, tmp_path, 10, 4, seed=83)
    away = str(tmp_path / "away")
    os.mkdir(away)
    sds = len(dat) // 10
    recs = _record_chunks(dat, live, sds, 10)
    path = base + ec.ToExt(5)
    full = open(path, "rb").read()
    half = len(full) // 2
    os.truncate(path, half)
    try:
        out = _read_with(ec, base, away, (0,), live)
    finally:
        open(path, "wb").write(full)
    both = 0
    for r, (key, want, chunks) in zip(out, recs):
        n = sum(1 for c in chunks if c[0] == 0 or (c[0] == 5 and c[1] + c[2] > half))
        assert r["status"] == "SWEC_OK" and (r["bytes"] == want).all(), (key, r["status"])
        assert r["recovered_intervals"] == n, (key, r["recovered_intervals"], n)
        both += any(c[0] == 0 and c[1] + c[2] > half for c in chunks)
    assert both > 0 and any(c[0] == 0 and c[1] + c[2] <= half for _, _, cs in recs for c in cs)


# ---------------------------------------------------------------- a volume just over one large row

GIB, MIB = 1 << 30, 1 << 20
# (needle id, .dat offset, Size): across the first 1 GiB block border of every large block, 3 MiB ones at the 3rd and
# 7th (their part after the border is one interval over the packed limit, so it streams), 5 MiB inside block 5, across
# the large→small seam, inside and across the 1 MiB blocks of the small row, and a last record whose read (GetActualSize
# applied twice) runs into the row's zero padding.  Gaps keep every read clear of the next record.
LARGE_RECORDS = ([(1, 8, 3000)] + [(1 + i, i * GIB - (12288 if i in (3, 7) else 1000 + 8 * i), 3 * MIB if i in (3, 7) else 10000 + i)
                                   for i in range(1, 10)]
                 + [(11, 5 * GIB + 100 * MIB, 5 * MIB), (12, 10 * GIB - 7000, 20000), (13, 10 * GIB + 64 * 1024, 900 * 1024),
                    (14, 10 * GIB + MIB - 504, 3000), (15, 10 * GIB + 2 * MIB - 8192, 10000)])
# on the same shard files: a record whose read runs 24 bytes past the end of the last row, i.e. past the shard files
PAST_END = (16, 10 * GIB + 10 * MIB - 8 - 1032, 1000)


def _actual(size):
    return rn.get_actual_size(size, 3)


def _chunks(sds, off, n):
    out = []
    for iv in rn.locate_data(GIB, MIB, sds, off, n, 10):
        sid, soff = rn.interval_to_shard(iv, GIB, MIB, 10)
        out.append((sid, soff, iv[2]))
    return out


def _write_index(base, records):
    dat_size = max(off + _actual(size) for _, off, size in records)
    open(base + ".ecx", "wb").write(b"".join(rn._entry(k, off // 8, size) for k, off, size in sorted(records)))
    json.dump({"version": 3, "datFileSize": str(dat_size), "ecShardConfig": {"dataShards": 10, "parityShards": 4}},
              open(base + ".vif", "w"))
    return dat_size


@pytest.fixture(scope="module")
def large_row_volume(tmp_path_factory):
    """Shard files of 1 GiB + 1 MiB holding only the records' bytes and, for every column they touch, the parity of that
    column (columns of zeros encode to zeros).  Written sparse: a few MiB on a filesystem that keeps holes, up to the
    files' 14 GiB on one that allocates them."""
    from oracle import pyoracle
    d = tmp_path_factory.mktemp("large_row")
    st = os.statvfs(d)
    if st.f_bavail * st.f_frsize < 16 * GIB:
        pytest.skip("the temporary directory has less than 16 GiB free for 14 shard files of 1 GiB + 1 MiB")
    return _lay_down_large_row(str(d / "5"), pyoracle)


def _lay_down_large_row(base, pyoracle):
    """Writes the sparse shard files of LARGE_RECORDS and PAST_END at base; returns (base, record bytes by id)."""
    rng = np.random.default_rng(0x1A26E)
    records = LARGE_RECORDS + [PAST_END]
    dat_size = max(off + _actual(size) for _, off, size in LARGE_RECORDS)
    shard_size = rn.expected_shard_size(dat_size)
    assert shard_size == GIB + MIB == rn.expected_shard_size(PAST_END[1] + _actual(PAST_END[2]))
    files = [open(base + ".ec%02d" % i, "w+b") for i in range(14)]
    contents, columns = {}, []
    try:
        for f in files:
            f.truncate(shard_size)
        for key, off, size in records:
            body = rng.integers(0, 256, _actual(size), dtype=np.uint8)
            contents[key] = body
            pos = 0
            for sid, soff, n in _chunks(dat_size // 10, off, len(body)):
                files[sid].seek(soff)
                files[sid].write(body[pos:pos + n].tobytes())
                columns.append((soff, soff + n))
                pos += n
        columns.sort()
        merged = [list(columns[0])]
        for a, b in columns[1:]:
            if a <= merged[-1][1]:
                merged[-1][1] = max(merged[-1][1], b)
            else:
                merged.append([a, b])
        for a, b in merged:
            data = []
            for f in files[:10]:
                f.seek(a)
                data.append(np.frombuffer(f.read(b - a), dtype=np.uint8).copy())
            for f, p in zip(files[10:], pyoracle.encode(10, 4, data)):
                f.seek(a)
                f.write(p.tobytes())
    finally:
        for f in files:
            f.close()
    return base, contents


def _expected_large(contents, key, size):
    want = _actual(_actual(size))
    return np.concatenate([contents[key], np.zeros(want - _actual(size), dtype=np.uint8)])


@pytest.mark.gpu
def test_degraded_needle_reads_just_over_one_large_row(cuda, swec, options, large_row_volume):
    """A 10 GiB + 2 MiB RS(10,4) volume (one large row of 1 GiB blocks, one small row of 1 MiB blocks that is mostly zero
    padding) with its datFileSize in .vif, read healthy, with 1, 2 and 4 data shards lost and with all parity lost:
    every record equals its bytes followed by the zero padding the double GetActualSize reads, and recovered_intervals
    equals its chunks (rs_numpy.locate_data over the large / small geometry) on lost data shards.  Some recovered
    intervals are over the packed limit and stream.

    Then the same shard files with a last record whose read runs 24 bytes past the end of the last row: the reference
    reads that interval short, from its own shard and from every other one (EcVolumeShard.ReadAt and the recovery
    count only full reads, store_ec.go:407-422,482-560), so ReadEcShardNeedle fails for it: SWEC_ERR_TOO_FEW_SHARDS,
    healthy or degraded, and every other record reads as before."""
    ec = swec.erasure_coding
    base, contents = large_row_volume
    away = os.path.join(os.path.dirname(base), "away")          # renames stay on the shard files' filesystem
    os.makedirs(away, exist_ok=True)
    dat_size = _write_index(base, LARGE_RECORDS)
    vol = ec.EcVolume(base, device=-1)
    sds = vol.info()["shard_dat_size"]
    vol.close()
    assert sds == dat_size // 10 and sds // GIB == 1
    expect = {key: (_expected_large(contents, key, size), _chunks(sds, off, _actual(_actual(size))))
              for key, off, size in LARGE_RECORDS}
    shards_of = {key: {c[0] for c in ch} for key, (_, ch) in expect.items()}
    assert all(shards_of[1 + i] == {i - 1, i} for i in range(1, 10))    # every 1 GiB border of the large row
    assert shards_of[12] == {9, 0}                                       # the seam: block 9 of the large row → small block 0
    assert any(c[1] >= GIB for c in expect[12][1]) and any(c[1] < GIB for c in expect[12][1])
    streamed = 0
    live = [(key, off, size) for key, off, size in LARGE_RECORDS]
    for lost in [(), (0,), (9,), (3, 4), (0, 9), (0, 1, 2, 3), (6, 7, 8, 9), (2, 5, 7, 8), (10, 11, 12, 13)]:
        out = _read_with(ec, base, away, lost, live)
        for r, (key, off, size) in zip(out, live):
            want, chunks = expect[key]
            gone = [c for c in chunks if c[0] in lost]
            assert r["status"] == "SWEC_OK", (lost, key, r["status"])
            assert r["offset"] == off and r["n_bytes"] == len(want) and (r["bytes"] == want).all(), (lost, key)
            assert r["recovered_intervals"] == len(gone), (lost, key, r["recovered_intervals"], len(gone))
            streamed += sum(1 for c in gone if c[2] > PACKED_LIMIT)
    assert streamed >= 3

    _write_index(base, LARGE_RECORDS + [PAST_END])
    key, off, size = PAST_END
    chunks = _chunks(sds, off, _actual(_actual(size)))
    assert chunks[-1][0] == 0 and chunks[-1][1] == GIB + MIB            # the read's last interval lies past the files
    for lost in [(), (0,), (9,)]:
        out = _read_with(ec, base, away, lost, live + [PAST_END])
        assert out[-1]["status"] == "SWEC_ERR_TOO_FEW_SHARDS", (lost, out[-1]["status"])
        for r, (k, o, s) in zip(out, live):
            want, ch = expect[k]
            assert r["status"] == "SWEC_OK" and (r["bytes"] == want).all(), (lost, k)
            assert r["recovered_intervals"] == sum(1 for c in ch if c[0] in lost), (lost, k)
