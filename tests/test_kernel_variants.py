"""Every launch shape and instruction mix of the matrix-apply kernels against the CPU oracle.

All parity bytes come from one templated Horner body (`swec_horner_body`, device_common.cuh) and the table and byte
kernels behind it; the engine picks the instantiation from the tuning options and the call's shape.  Every
instantiation computes the same bytes, so each case here checks the bytes against the oracle (`oracle.encode`,
`rs_numpy.apply_rows`) and, through torch.profiler, which kernel computed them: a dispatch mix-up shows only in the
kernel name.  Columns are independent, so one oracle result over the longest stream serves every shorter run as a
prefix.  Lengths are derived from the device's SM count: several grid passes, a last tile in which only some threads
are live, and a tail for the byte kernel.

CPU part: the ledger (the kernel instantiations in libswec.so are exactly the ones the GPU part covers) and an NVRTC
compile of every specialised-kernel key the GPU part uses (which also fills the suite's cubin cache)."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import sys
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))

SHAPES = [(128, 1), (128, 2), (256, 1), (256, 2), (512, 1), (512, 2)]   # enc_threads × enc_unroll
POWER_MODES = (1, 2)                                                      # boost, low-power step
ENCODE_CTAS = (0, 1, 64)                                                  # derived, several passes, one CTA per tile
RECON_PATTERNS = [(i,) for i in range(14)] + [(0, 1, 2, 3)]               # the compiled-in reconstruct matrices
BLOCKS = (16, 48, 4112, 65536)                                            # block_vecs 1 (shift), 3 and 257 (division), 4096
SENTINEL = 0xA5

# the options every case starts from and is returned to (kernels.cu, engine.cc: the documented defaults)
DEFAULTS = {"enc_threads": 512, "enc_unroll": 2, "ctas_per_sm": 0, "xt_variant": 0, "power_mode": 1, "use_aot": 1,
            "jit": 1, "jit_min_bytes": 64 << 20, "jit_share_powers": 0}

# what the GPU part checks by name; test_ledger_matches_the_library holds the library to exactly this set
COVERED = ({("rs10x4_encode", t, u, b, lp) for t, u in SHAPES for b in (False, True) for lp in (False, True)}
           | {("swec_aot_recon", ns, i) for ns in ("swec_aot_boost", "swec_aot_lowpower") for i in range(len(RECON_PATTERNS))}
           | {("swec_table_kernel", 0), ("swec_table_kernel", 10), ("swec_bytes_kernel",)})


# ---------------------------------------------------------------- kernel names

_BOOL = {"true": True, "false": False, "1": True, "0": False}


def kernel_id(name):
    """A kernel's identity from its mangled or demangled name, or None for kernels outside the matrix-apply family."""
    m = re.search(r"rs10x4_encodeILi(\d+)ELi(\d+)ELb([01])ELb([01])E", name) or \
        re.search(r"rs10x4_encode<(\d+), ?(\d+), ?(true|false|1|0), ?(true|false|1|0)>", name)
    if m:
        return ("rs10x4_encode", int(m[1]), int(m[2]), _BOOL[m[3]], _BOOL[m[4]])
    m = re.search(r"swec_aot_reconIN\d+(swec_aot_boost|swec_aot_lowpower)\d+SwecAotRecon(\d+)E", name) or \
        re.search(r"swec_aot_recon<(swec_aot_boost|swec_aot_lowpower)::SwecAotRecon(\d+)>", name)
    if m:
        return ("swec_aot_recon", m[1], int(m[2]))
    m = re.search(r"swec_table_kernel(?:ILi(\d+)E|<(\d+)>)", name)
    if m:
        return ("swec_table_kernel", int(m[1] or m[2]))
    for plain in ("swec_bytes_kernel", "swec_jit_flat", "swec_jit_blocked"):
        if plain in name:
            return (plain,)
    return None


def encode_id(threads, unroll, blocked, power_mode):
    return ("rs10x4_encode", threads, unroll, blocked, power_mode == 2)


class Launches:
    """The matrix-apply kernels launched inside the block, recorded with torch.profiler (CUDA activity).  `ids` is
    None when the profiler recorded no kernel at all (no CUPTI): then only the bytes can be checked."""

    def __init__(self, torch):
        self.torch = torch

    def __enter__(self):
        from torch.profiler import ProfilerActivity, profile
        self.torch.cuda.synchronize()
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.__enter__()
        return self

    def __exit__(self, *exc):
        self.torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        if exc[0] is not None:
            return False
        from torch.autograd import DeviceType
        names = [e.name for e in self.prof.events() if e.device_type == DeviceType.CUDA]
        self.ids = [k for k in map(kernel_id, names) if k is not None] if names else None
        return False


def no_names(context):
    warnings.warn(f"torch.profiler recorded no kernels (CUPTI unavailable?): kernel names of {context} not checked")


def assert_launched(rec, want, context):
    """The matrix-apply kernels of the block are exactly the set `want` (skipped when the profiler saw nothing)."""
    if rec.ids is None:
        no_names(context)
        return
    assert set(rec.ids) == set(want), (context, sorted(set(rec.ids)), sorted(want))


# ---------------------------------------------------------------- shapes derived from the device

def derived_ctas(threads, unroll):
    """encode_ctas_per_sm() at ctas_per_sm = 0 (kernels.cu)"""
    return max(1, (512 if unroll > 1 else 768) // threads)


def encode_long_vectors(sms, threads, unroll):
    """Two full grid passes of the derived launch, then a tile in which only some threads are live (with two slices,
    all threads' first slice and half the threads' second one)."""
    tile = threads * unroll
    partial = threads + threads // 2 if unroll == 2 else threads // 2
    return 2 * sms * derived_ctas(threads, unroll) * tile + partial


def blocked_rows(sms, block):
    """Large rows per test volume; the 64 KiB one spans two grid passes of every shape at ctas_per_sm = 1."""
    return {16: 5000, 48: 3000, 4112: 40, 65536: 2 * sms * 1024 // 4096 + 2}[block]


def table_residency(k):
    """CTAs per SM of the table kernel (launch_table_apply)"""
    smem = k * 4096
    return 4 if smem <= 56 * 1024 else (2 if smem <= 113 * 1024 else 1)


def table_len(sms, k):
    """two grid passes of the table kernel, a partial third and a 13-byte tail"""
    grid_pass = sms * table_residency(k) * 256
    return (2 * grid_pass + grid_pass // 2 + 37) * 16 + 13


def round_up(n, a=256):
    return (n + a - 1) // a * a


# ---------------------------------------------------------------- options

def set_options(L, **opts):
    for name, value in opts.items():
        assert L.swec_set_option(name.encode(), int(value)) == 0, (name, value, L.swec_last_error())


def reset_options(L):
    set_options(L, **DEFAULTS)


@pytest.fixture
def options(swec):
    """The library's options, back to the documented defaults afterwards (there is no getter)."""
    L = swec.lib()
    try:
        yield L
    finally:
        reset_options(L)


def jit_counts(L):
    c, h = C.c_uint64(0), C.c_uint64(0)
    L.swec_jit_stats(C.byref(c), C.byref(h), None, None)
    return c.value + h.value


# ---------------------------------------------------------------- the specialised-kernel keys

def nvrtc_matrices(ec):
    """The run-time matrices of the NVRTC cases, taken from the product's own generator and decode plan."""
    rng = np.random.default_rng(0x5EC)
    e10, e24 = ec.Encoder(10, 4, device=0), ec.Encoder(24, 8, device=0)
    try:
        _, outs, lost = e10.reconstruct_matrix([0] * 4 + [1] * 10)
        assert outs == [0, 1, 2, 3]
        return {"rs10x4_parity": e10.matrix()[10:].copy(), "lost_0_3": lost, "rs24x8_parity": e24.matrix()[24:].copy(),
                "apply_1x32": rng.integers(1, 256, (1, 32), dtype=np.uint8),
                "toggle_2x7": rng.integers(1, 256, (2, 7), dtype=np.uint8)}
    finally:
        e10.close()
        e24.close()


def variant_options(xt, share_powers):
    # xt 0 is the boost step, which power_mode 1 keeps; xt 1-3 override the power policy
    return {"xt_variant": xt, "power_mode": 1, "jit_share_powers": share_powers}


def nvrtc_cases():
    """(matrix, options) of every NVRTC key the GPU part compiles, in the order it compiles them."""
    cases = [("rs10x4_parity", dict(enc_threads=t, enc_unroll=u, **variant_options(xt, sp)))
             for t, u in SHAPES for xt in range(4) for sp in (0, 1)]
    for name in ("lost_0_3", "rs24x8_parity", "apply_1x32"):
        cases += [(name, dict(enc_threads=t, enc_unroll=u, **variant_options(0, 0))) for t, u in SHAPES]
        cases += [(name, dict(enc_threads=512, enc_unroll=2, **variant_options(xt, sp)))
                  for xt in range(4) for sp in (0, 1) if (xt, sp) != (0, 0)]
    return cases


TOGGLES = [("enc_threads", 256), ("enc_unroll", 1), ("xt_variant", 1), ("jit_share_powers", 1), ("power_mode", 2)]


# ================================================================ CPU part

def test_kernel_id_reads_both_spellings():
    assert kernel_id("_ZN4swec13rs10x4_encodeILi256ELi1ELb1ELb0EEEv15SwecApplyParams") == \
        kernel_id("void swec::rs10x4_encode<256, 1, true, false>(SwecApplyParams)") == ("rs10x4_encode", 256, 1, True, False)
    assert kernel_id("_ZN4swec14swec_aot_reconIN17swec_aot_lowpower13SwecAotRecon9EEEv15SwecApplyParams") == \
        kernel_id("void swec::swec_aot_recon<swec_aot_lowpower::SwecAotRecon9>(SwecApplyParams)") == \
        ("swec_aot_recon", "swec_aot_lowpower", 9)
    assert kernel_id("void swec::swec_table_kernel<10>(SwecApplyParams, unsigned int const*, int, int)") == \
        kernel_id("_ZN4swec17swec_table_kernelILi10EEEv15SwecApplyParamsPKjii") == ("swec_table_kernel", 10)
    assert kernel_id("swec_jit_blocked") == ("swec_jit_blocked",) and kernel_id("void at::native::fill_kernel") is None


def test_ledger_matches_the_library(swec):
    """The matrix-apply instantiations compiled into libswec.so are exactly the ones the GPU part checks by name: a
    new instantiation fails here until a test launches it."""
    from seaweedfs_b200 import _native
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("no CUDA toolkit")
    out = subprocess.run([cuobjdump, "-symbols", _native.library_path()], capture_output=True, text=True,
                         check=True).stdout
    found = {kernel_id(ln.split()[-1]) for ln in out.splitlines() if "STT_FUNC" in ln and "STO_ENTRY" in ln}
    found.discard(None)
    assert found == COVERED, {"not covered": sorted(found - COVERED), "not in the library": sorted(COVERED - found)}


def test_nvrtc_compiles_every_key_and_share_powers_lowers_the_steps(swec, options):
    """swec_debug_jit_compile of every key the GPU part launches (this fills the suite's cubin cache).  Shared power
    chains lower the multiply-by-2 steps of the two matrices the GPU part relies on for them: RS(10,4) encode 24 -> 20,
    data shards 0-3 lost 27 -> 21.  Other options never change the step count."""
    L = options
    mats = nvrtc_matrices(swec.erasure_coding)
    steps = {}
    for name, opts in nvrtc_cases() + [("toggle_2x7", {})] + [("toggle_2x7", {o: v}) for o, v in TOGGLES]:
        reset_options(L)
        set_options(L, **opts)
        rows = np.ascontiguousarray(mats[name])
        size, st, xors = C.c_size_t(0), C.c_int(0), C.c_int(0)
        rc = L.swec_debug_jit_compile(rows.shape[0], rows.shape[1], rows.ctypes.data, C.byref(size), C.byref(st),
                                      C.byref(xors))
        if rc == -8 and b"not available" in L.swec_last_error():
            pytest.skip("NVRTC not installed here")
        assert rc == 0 and size.value > 1000, (name, opts, L.swec_last_error())
        steps.setdefault((name, opts.get("jit_share_powers", 0)), set()).add(st.value)
    assert all(len(v) == 1 for v in steps.values()), steps
    one = {k: next(iter(v)) for k, v in steps.items()}
    assert (one[("rs10x4_parity", 0)], one[("rs10x4_parity", 1)]) == (24, 20)
    assert (one[("lost_0_3", 0)], one[("lost_0_3", 1)]) == (27, 21)
    for name in ("rs24x8_parity", "apply_1x32", "toggle_2x7"):
        assert one[(name, 1)] <= one[(name, 0)], (name, one)
    print(json.dumps({f"{n} share_powers={s}": v for (n, s), v in one.items()}))


# ================================================================ GPU part

def _dev(torch, arr):
    return torch.from_numpy(np.ascontiguousarray(arr)).cuda()


def _stream(torch):
    return torch.cuda.current_stream().cuda_stream


def _outputs(torch, rows, n):
    return torch.full((rows, round_up(n + 64)), SENTINEL, dtype=torch.uint8, device="cuda")


def _check(torch, out, want, n, context):
    """out[:, :n] is the oracle's and the bytes after it are untouched"""
    r = want.shape[0]
    assert torch.equal(out[:r, :n], want[:, :n]), context
    assert bool((out[:r, n:] == SENTINEL).all()), (context, "write past the end")


def _restripe(torch, data, rows, block):
    """A volume of `rows` large rows of `block`-byte blocks whose shard i is data[i][:rows*block], so that its parity is
    the flat parity's prefix of rows*block bytes."""
    k = data.shape[0]
    return data[:, :rows * block].reshape(k, rows, block).transpose(0, 1).contiguous().reshape(-1)


@pytest.fixture(scope="module")
def sms(cuda):
    return cuda.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def encode_pool(cuda, oracle, sms):
    """10 data streams long enough for every flat and blocked case, their oracle parity, and the blocked volumes."""
    torch = cuda
    n = round_up(max([encode_long_vectors(sms, t, u) * 16 + 13 for t, u in SHAPES] +
                     [blocked_rows(sms, b) * b for b in BLOCKS]) + 64)
    rng = np.random.default_rng(0x10AE)
    data = [rng.integers(0, 256, n, dtype=np.uint8) for _ in range(10)]
    d, w = _dev(torch, np.stack(data)), _dev(torch, np.stack(oracle.encode(10, 4, data)))
    vols = {b: _restripe(torch, d, blocked_rows(sms, b), b) for b in BLOCKS}
    return d, w, vols


@pytest.mark.gpu
@pytest.mark.parametrize("threads,unroll", SHAPES)
def test_aot_encode_every_shape(cuda, swec, options, encode_pool, sms, threads, unroll):
    """The 24 RS(10,4) encode instantiations: each (threads, unroll) at power_mode 1 and 2 and ctas_per_sm 0 (derived),
    1 (many grid passes) and 64 (one CTA per tile).  Flat: 16 B, one exact tile, and two grid passes plus a partial
    tile plus a 13-byte tail; blocked: large blocks of 16, 48, 4112 and 65536 bytes over several rows, the 64 KiB ones
    over two grid passes at ctas_per_sm 1."""
    torch, L = cuda, options
    d, w, vols = encode_pool
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    s = _stream(torch)
    lengths = [16, threads * unroll * 16, encode_long_vectors(sms, threads, unroll) * 16 + 13]
    try:
        for pm in POWER_MODES:
            for ctas in ENCODE_CTAS:
                set_options(L, enc_threads=threads, enc_unroll=unroll, power_mode=pm, ctas_per_sm=ctas)
                ctx = f"{threads}x{unroll} power_mode={pm} ctas_per_sm={ctas}"
                with Launches(torch) as rec:
                    for n in lengths:
                        out = _outputs(torch, 4, n)
                        enc.encode_device([d[i].data_ptr() for i in range(10)], [out[p].data_ptr() for p in range(4)], n, s)
                        _check(torch, out, w, n, (ctx, "flat", n))
                    for block in BLOCKS:
                        rows = blocked_rows(sms, block)
                        out = _outputs(torch, 4, rows * block)
                        enc.encode_volume_device(vols[block].data_ptr(), rows * 10 * block, [out[p].data_ptr() for p in range(4)],
                                                 s, large_block=block, small_block=16)
                        _check(torch, out, w, rows * block, (ctx, "blocked", block))
                assert_launched(rec, {encode_id(threads, unroll, False, pm), encode_id(threads, unroll, True, pm),
                                      ("swec_bytes_kernel",)}, ctx)
    finally:
        enc.close()


@pytest.fixture(scope="module")
def table_pool(cuda, sms):
    """32 input streams and a random 12×32 matrix; the 4×K and r×K cases use its leading rows and columns."""
    torch = cuda
    n = round_up(max(table_len(sms, k) for k in range(1, 33)) + 64)
    rng = np.random.default_rng(0x7AB1E)
    x = rng.integers(0, 256, (32, n), dtype=np.uint8)
    m = rng.integers(0, 256, (12, 32), dtype=np.uint8)
    return x, _dev(torch, x), m


def _apply(enc, torch, rows, ins, outs, n):
    enc.apply_device(rows, [t.data_ptr() for t in ins], [t.data_ptr() for t in outs], n, _stream(torch))


def _table_id(k):
    return ("swec_table_kernel", 10 if k == 10 else 0)


@pytest.mark.gpu
def test_table_and_byte_kernels_every_k(cuda, swec, options, table_pool, sms):
    """jit = 0: a 4×K matrix for K = 1…32, r = 1…4 as row prefixes, over two grid passes of the table kernel (4, 2 or 1
    CTAs per SM by K), a partial pass and a 13-byte tail; then the same matrices on pointers offset by 1…15 bytes,
    longer than one pass of the byte kernel, with the bytes either side of every output untouched."""
    from oracle import rs_numpy as rn
    torch, L = cuda, options
    x, xd, m = table_pool
    set_options(L, jit=0)
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    n_unaligned = sms * 8 * 256 + 4099
    acc = np.zeros((4, x.shape[1]), dtype=np.uint8)
    try:
        for k in range(1, 33):
            for r in range(4):                       # the oracle for K columns: that of K-1 plus column K-1's terms
                acc[r] ^= rn.MUL[int(m[r, k - 1])][x[k - 1]]
            want = _dev(torch, acc)
            n = table_len(sms, k)
            ins = [xd[i] for i in range(k)]
            with Launches(torch) as rec:
                for r in range(1, 5):
                    out = _outputs(torch, 4, n)
                    _apply(enc, torch, m[:r, :k], ins, [out[p] for p in range(r)], n)
                    _check(torch, out[:r], want[:r], n, ("K", k, "r", r))
                    assert bool((out[r:] == SENTINEL).all()), ("K", k, "r", r, "rows past r written")
            assert_launched(rec, {_table_id(k), ("swec_bytes_kernel",)}, f"table K={k}")
            with Launches(torch) as rec:
                for off in range(1, 16):
                    back_in = torch.zeros((k, n_unaligned + 32), dtype=torch.uint8, device="cuda")
                    back_in[:, off:off + n_unaligned] = xd[:k, :n_unaligned]
                    back_out = torch.full((4, n_unaligned + 32), SENTINEL, dtype=torch.uint8, device="cuda")
                    _apply(enc, torch, m[:4, :k], [back_in[i, off:] for i in range(k)],
                           [back_out[p, off:] for p in range(4)], n_unaligned)
                    assert torch.equal(back_out[:, off:off + n_unaligned], want[:, :n_unaligned]), ("K", k, "offset", off)
                    assert bool((back_out[:, :off] == SENTINEL).all()) and \
                        bool((back_out[:, off + n_unaligned:] == SENTINEL).all()), ("K", k, "offset", off, "guard")
            assert_launched(rec, {("swec_bytes_kernel",)}, f"unaligned K={k}")
    finally:
        enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("k", [10, 32])
def test_table_kernels_more_than_four_rows(cuda, swec, options, table_pool, sms, k):
    """jit = 0: r = 5…12 rows at K = 10 and 32 take one table launch per group of four rows; aligned over two grid
    passes plus a tail, and on pointers offset by 1…15 bytes."""
    from oracle import rs_numpy as rn
    torch, L = cuda, options
    x, xd, m = table_pool
    set_options(L, jit=0)
    n = table_len(sms, k)
    n_unaligned = sms * 8 * 256 + 4099
    want = _dev(torch, np.stack(rn.apply_rows(m[:, :k], list(x[:k, :n]))))
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    ins = [xd[i] for i in range(k)]
    try:
        with Launches(torch) as rec:
            for r in range(5, 13):
                out = _outputs(torch, 12, n)
                _apply(enc, torch, m[:r, :k], ins, [out[p] for p in range(r)], n)
                _check(torch, out[:r], want[:r], n, ("K", k, "r", r))
                assert bool((out[r:] == SENTINEL).all()), ("K", k, "r", r, "rows past r written")
        assert_launched(rec, {_table_id(k), ("swec_bytes_kernel",)}, f"table K={k} r>4")
        for off in range(1, 16):
            back_in = torch.zeros((k, n_unaligned + 32), dtype=torch.uint8, device="cuda")
            back_in[:, off:off + n_unaligned] = xd[:k, :n_unaligned]
            back_out = torch.full((12, n_unaligned + 32), SENTINEL, dtype=torch.uint8, device="cuda")
            _apply(enc, torch, m[:, :k], [back_in[i, off:] for i in range(k)], [back_out[p, off:] for p in range(12)],
                   n_unaligned)
            assert torch.equal(back_out[:, off:off + n_unaligned], want[:, :n_unaligned]), ("K", k, "offset", off)
            assert bool((back_out[:, :off] == SENTINEL).all()) and \
                bool((back_out[:, off + n_unaligned:] == SENTINEL).all()), ("K", k, "offset", off, "guard")
    finally:
        enc.close()


@pytest.mark.gpu
def test_aot_reconstruct_every_pattern(cuda, swec, oracle, options, sms):
    """The 15 compiled-in reconstruct kernels in both instruction mixes (power_mode 1 and 2), over two grid passes of
    the lightest launch (S·2·1024 vectors) plus a partial one plus a tail, compared on the device with the original
    shards."""
    torch, L = cuda, options
    nvec = 2 * sms * 2 * 1024 + 1024 + 512 + 7
    n = nvec * 16 + 13
    rng = np.random.default_rng(0xAEC0)
    data = [rng.integers(0, 256, n, dtype=np.uint8) for _ in range(10)]
    full = torch.full((14, round_up(n)), SENTINEL, dtype=torch.uint8, device="cuda")   # 16-byte aligned rows
    full[:, :n] = _dev(torch, np.stack(data + oracle.encode(10, 4, data)))
    aot = C.c_int(0)
    L.swec_jit_stats(None, None, C.byref(aot), None)
    assert aot.value == len(RECON_PATTERNS)
    enc = swec.erasure_coding.Encoder(10, 4, device=0)
    try:
        for pm in POWER_MODES:
            set_options(L, power_mode=pm)
            ns = "swec_aot_boost" if pm == 1 else "swec_aot_lowpower"
            seen = set()
            for lost in RECON_PATTERNS:
                work = full.clone()
                work[list(lost)] = SENTINEL
                with Launches(torch) as rec:
                    enc.reconstruct_device([work[i].data_ptr() for i in range(14)], [i not in lost for i in range(14)], n,
                                           False, _stream(torch))
                assert torch.equal(work, full), (pm, lost)
                if rec.ids is None:
                    no_names(f"reconstruct {lost}")
                else:
                    recon = [i for i in rec.ids if i[0] == "swec_aot_recon"]
                    assert len(recon) == 1 and recon[0][1] == ns, (pm, lost, rec.ids)
                    assert set(rec.ids) == {recon[0], ("swec_bytes_kernel",)}, (pm, lost, rec.ids)
                    seen.add(recon[0])
            if seen:
                assert len(seen) == len(RECON_PATTERNS), (pm, sorted(seen))   # one kernel of its own per pattern
    finally:
        enc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [80_011, 3 * 4096 + 5])
def test_verify_counts_differing_vectors(cuda, swec, oracle, tmp_path, monkeypatch, n):
    """verify_ec_files with 4 KiB slots on shards whose length is not a multiple of 16: mismatched_vectors is the
    number of differing 16-byte vectors (include/swec.h), the partial last vector counting once."""
    ec = swec.erasure_coding
    monkeypatch.setenv("SWEC_FILE_CHUNK", "4096")
    rng = np.random.default_rng(n)
    data = [rng.integers(0, 256, n, dtype=np.uint8) for _ in range(10)]
    shards = data + oracle.encode(10, 4, data)
    base = str(tmp_path / "7")
    last = n - n % 16                                 # first byte of the partial last vector
    damage = {10: [100 * 16 + 3, 100 * 16 + 9, last - 1, last],    # two bytes in one vector; either side of the last edge
              11: [500 * 16 - 1, 500 * 16],                         # either side of a vector boundary
              12: list(range(4096 - 16, 4096)) + [8192],            # a whole vector before a slot edge, one after another
              13: [last, n - 1]}                                    # the partial last vector
    stored = [s.copy() for s in shards]
    for p, offs in damage.items():
        for off in offs:
            stored[p][off] ^= 0x5A
    for i, s in enumerate(stored):
        s.tofile(base + ec.ToExt(i))
    want = [len(np.unique(np.nonzero(stored[p] != shards[p])[0] // 16)) for p in range(10, 14)]
    assert all(want)
    assert ec.verify_ec_files(base) == (False, want)
    for i, s in enumerate(shards):
        s.tofile(base + ec.ToExt(i))
    assert ec.verify_ec_files(base) == (True, [0, 0, 0, 0])


# ---------------------------------------------------------------- NVRTC kernels, in a process of their own

def _nvrtc_child():
    """Runs in a fresh process, so that every key is new to the in-process caches and costs exactly one compile or one
    disk-cache hit.  Prints RESULT <json>: one record per case."""
    import torch
    import seaweedfs_b200
    from oracle import pyoracle as po, rs_numpy as rn
    from seaweedfs_b200 import erasure_coding as ec
    L = seaweedfs_b200.lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    mats = nvrtc_matrices(ec)
    s = torch.cuda.current_stream().cuda_stream
    n = round_up(max(encode_long_vectors(sms, t, u) * 16 + 13 for t, u in SHAPES) + 64)
    rng = np.random.default_rng(0x717)
    x = rng.integers(0, 256, (32, n), dtype=np.uint8)
    xd = _dev(torch, x)
    want = {"rs10x4_parity": po.encode(10, 4, list(x[:10])), "lost_0_3": list(x[:4]),
            "rs24x8_parity": po.encode(24, 8, list(x[:24])), "apply_1x32": rn.apply_rows(mats["apply_1x32"], list(x)),
            "toggle_2x7": rn.apply_rows(mats["toggle_2x7"], list(x[:7]))}
    want = {k: _dev(torch, np.stack(v)) for k, v in want.items()}
    parity10 = _dev(torch, np.stack(po.encode(10, 4, list(x[:10]))))
    encs = {"rs10x4_parity": ec.Encoder(10, 4, 0), "lost_0_3": ec.Encoder(10, 4, 0),
            "rs24x8_parity": ec.Encoder(24, 8, 0), "apply_1x32": ec.Encoder(10, 4, 0), "toggle_2x7": ec.Encoder(10, 4, 0)}
    blocks = {"rs10x4_parity": (10, 4), "rs24x8_parity": (24, 8)}
    vols = {(name, b): _restripe(torch, xd[:k], 3 if b == 4112 else 2, b) for name, (k, m) in blocks.items()
            for b in (4112, 65536)}
    out = []

    def flat(name, nbytes):
        e, w = encs[name], want[name]
        o = _outputs(torch, w.shape[0], nbytes)
        optr = [o[p].data_ptr() for p in range(w.shape[0])]
        if name == "lost_0_3":                       # the rebuilt data shards 0-3 are the outputs
            shards = optr + [xd[i].data_ptr() for i in range(4, 10)] + [parity10[p].data_ptr() for p in range(4)]
            e.reconstruct_device(shards, [0] * 4 + [1] * 10, nbytes, False, s)
        elif name in blocks:
            e.encode_device([xd[i].data_ptr() for i in range(blocks[name][0])], optr, nbytes, s)
        else:
            rows = mats[name]
            e.apply_device(rows, [xd[i].data_ptr() for i in range(rows.shape[1])], optr, nbytes, s)
        torch.cuda.synchronize()
        return torch.equal(o[:, :nbytes], w[:, :nbytes]) and bool((o[:, nbytes:] == SENTINEL).all())

    def blocked(name):
        k, m = blocks[name]
        oks = []
        for b in (4112, 65536):
            rows = 3 if b == 4112 else 2
            o = _outputs(torch, m, rows * b)
            encs[name].encode_volume_device(vols[(name, b)].data_ptr(), rows * k * b, [o[p].data_ptr() for p in range(m)],
                                            s, large_block=b, small_block=16)
            torch.cuda.synchronize()
            oks.append(torch.equal(o[:, :rows * b], want[name][:, :rows * b]) and bool((o[:, rows * b:] == SENTINEL).all()))
        return all(oks)

    def run(name, opts, label):
        reset_options(L)
        set_options(L, jit_min_bytes=1, use_aot=0, **opts)
        t, u = opts.get("enc_threads", 512), opts.get("enc_unroll", 2)
        c0 = jit_counts(L)
        with Launches(torch) as rec:
            ok = flat(name, encode_long_vectors(sms, t, u) * 16 + 13)
        c1 = jit_counts(L)
        names = rec.ids
        if name in blocks:
            with Launches(torch) as rec:
                ok = blocked(name) and ok
            names = None if names is None or rec.ids is None else names + rec.ids
        rec_out = {"case": label, "matrix": name, "options": opts, "ok": bool(ok), "first_cost": c1 - c0,
                   "later_cost": jit_counts(L) - c1, "ids": sorted(set(names)) if names is not None else None}
        out.append(rec_out)
        return rec_out

    try:
        for name, opts in nvrtc_cases():
            run(name, opts, "key")
        run("toggle_2x7", {}, "toggle base")
        for opt, val in TOGGLES:
            run("toggle_2x7", {opt: val}, "toggle")
            run("toggle_2x7", {}, "toggle back")
    finally:
        reset_options(L)
    print("RESULT " + json.dumps(out))


@pytest.fixture(scope="module")
def nvrtc_results(cuda):
    env = dict(os.environ)
    env.pop("SWEC_NO_JIT", None)
    code = f"import sys; sys.path[:0] = [{ROOT!r}, {HERE!r}]; import test_kernel_variants as t; t._nvrtc_child()"
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(next(ln for ln in r.stdout.splitlines() if ln.startswith("RESULT "))[7:])


def _jit_ids(name):
    return {("swec_jit_flat",), ("swec_bytes_kernel",)} | ({("swec_jit_blocked",)} if name in ("rs10x4_parity", "rs24x8_parity") else set())


@pytest.mark.gpu
def test_nvrtc_every_key(nvrtc_results):
    """jit_min_bytes = 1, use_aot = 0: RS(10,4) parity at every shape × xt_variant 0-3 × jit_share_powers 0/1, flat and
    blocked (block_vecs 257 and 4096); the data-shards-0-3 reconstruct, RS(24,8) encode (flat and blocked) and a random
    1×32 apply at every shape, and every variant × share_powers at 512×2.  Each key costs exactly one compile or one
    disk-cache hit, and its later calls none."""
    keys = [r for r in nvrtc_results if r["case"] == "key"]
    assert len(keys) == len(nvrtc_cases())
    bad = [r for r in keys if not r["ok"] or r["first_cost"] != 1 or r["later_cost"] != 0 or
           (r["ids"] is not None and {tuple(i) for i in r["ids"]} != _jit_ids(r["matrix"]))]
    assert not bad, bad[:5]
    if keys[0]["ids"] is None:
        no_names("the NVRTC cases")


@pytest.mark.gpu
def test_nvrtc_every_option_in_the_key_makes_a_new_kernel(nvrtc_results):
    """On a matrix already compiled, changing enc_threads, enc_unroll, xt_variant, jit_share_powers or power_mode
    compiles (or loads) a kernel of its own, and changing it back finds the first one in the cache again."""
    tog = [r for r in nvrtc_results if r["case"].startswith("toggle")]
    assert [r["case"] for r in tog] == ["toggle base"] + ["toggle", "toggle back"] * len(TOGGLES)
    assert all(r["ok"] for r in tog), tog
    assert tog[0]["first_cost"] == 1
    costs = {next(iter(r["options"])): r["first_cost"] for r in tog if r["case"] == "toggle"}
    assert costs == {opt: 1 for opt, _ in TOGGLES}, costs
    assert all(r["first_cost"] == 0 for r in tog if r["case"] == "toggle back"), tog
