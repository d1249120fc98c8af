"""CPU-only checks of the product's host side: libswec.so loads without a GPU, exports exactly
what include/swec.h declares, its matrices and layout arithmetic agree with the oracle, and compute
entry points fail loudly (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    text = open(os.path.join(ROOT, "include", "swec.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(swec_[a-z0-9_]+)\s*\(", text)))


def test_header_and_library_agree(swec):
    from seaweedfs_b200._native import PROTOTYPES, library_path
    names = declared_functions()
    assert len(names) >= 25
    exported = subprocess.run(["nm", "-D", "--defined-only", library_path()], check=True,
                              stdout=subprocess.PIPE, text=True).stdout
    exported = set(re.findall(r" T (swec_[a-z0-9_]+)", exported))
    assert set(names) == exported, (set(names) ^ exported)
    assert set(names) == set(PROTOTYPES)
    L = swec.lib()
    for n in names:
        assert getattr(L, n)


def test_library_needs_no_gpu_to_load(swec):
    out = subprocess.run(["ldd", swec.library_path()], check=True, stdout=subprocess.PIPE, text=True).stdout
    assert "libcuda.so" not in out and "libnvrtc" not in out and "not found" not in out


def test_library_is_sm90a_only(swec):
    out = subprocess.run(["cuobjdump", "--list-elf", swec.library_path()], stdout=subprocess.PIPE, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_strerror_and_version(swec):
    L = swec.lib()
    assert b"sm_90a" in L.swec_version()
    assert L.swec_strerror(0) == b"ok"
    assert b"CPU fallback" in L.swec_strerror(-7)


@pytest.mark.parametrize("k,m", [(10, 4), (5, 5), (3, 2), (12, 4), (20, 12), (1, 1), (16, 16)])
def test_generator_matches_oracle(swec, oracle, k, m):
    enc = swec.erasure_coding.Encoder(k, m, device=-1)
    assert (enc.matrix() == oracle.build_matrix(k, k + m)).all()


@pytest.mark.parametrize("bad", [(0, 4), (10, 0), (-1, 2), (30, 3), (32, 1)])
def test_encoder_rejects_bad_ratios(swec, bad):
    # reedsolomon.New → ErrInvShardNum ; SeaweedFS: ds+ps <= MaxShardCount (ec_encoder.go:81)
    with pytest.raises(swec.SwecError) as e:
        swec.erasure_coding.Encoder(bad[0], bad[1], device=-1)
    assert e.value.name == "SWEC_ERR_INVALID_ARG"


def test_reconstruct_matrix_matches_oracle(swec, kat):
    from oracle import rs_numpy as rn
    enc = swec.erasure_coding.Encoder(10, 4, device=-1)
    rng = np.random.default_rng(11)
    patterns = [[0, 1, 2, 3], [10, 11, 12, 13], [0, 1, 10, 11], [5], [13], [2, 7, 12]]
    patterns += [sorted(rng.choice(14, size=rng.integers(1, 5), replace=False).tolist()) for _ in range(40)]
    for erased in patterns:
        present = [i not in erased for i in range(14)]
        for data_only in (False, True):
            valid, missing, rows = rn.fused_reconstruct_rows(10, 4, present, data_only)
            ins, outs, got = enc.reconstruct_matrix(present, data_only)
            assert ins == valid and outs == missing and (got == rows).all()
    # SURVEY §8(c) worst case
    _, _, rows = enc.reconstruct_matrix([0, 0, 0, 0] + [1] * 10)
    assert rows[0].tolist() == [29, 239, 227, 16, 49, 195, 195, 48, 13, 12]
    with pytest.raises(swec.SwecError) as e:
        enc.reconstruct_matrix([0] * 5 + [1] * 9)
    assert e.value.name == "SWEC_ERR_TOO_FEW_SHARDS"


def test_layout_matches_oracle(swec, oracle, kat):
    ec = swec.erasure_coding
    for case in kat["K7"]:
        assert ec.LocateData(*case["args"]) == [tuple(iv) for iv in case["intervals"]]
    rng = np.random.default_rng(5)
    for _ in range(300):
        large = int(rng.choice([10000, 1 << 20, 1 << 30]))
        small = int(rng.choice([100, 4096, 1 << 20]))
        if small > large:
            continue
        dat = int(rng.integers(1, 40 * large))
        shard = ec.expected_shard_size(dat, 10, large, small)
        assert shard == oracle.expected_shard_size(dat, 10, large, small)
        off = int(rng.integers(0, dat))
        size = int(rng.integers(1, min(dat - off, 5 * small) + 1))
        want = oracle.locate_data(large, small, dat // 10, off, size)
        got = ec.locate_data(large, small, dat // 10, off, size)
        assert got == want
        for iv in got:
            from oracle import rs_numpy as rn
            assert ec.interval_to_shard(iv, large, small) == rn.interval_to_shard(iv, large, small)


def test_compute_fails_loudly_without_device(swec):
    ec = swec.erasure_coding
    enc = ec.Encoder(10, 4, device=-1)
    shards = [np.zeros(64, dtype=np.uint8) for _ in range(14)]
    with pytest.raises(swec.SwecError) as e:
        enc.encode(shards)
    assert e.value.name == "SWEC_ERR_NO_DEVICE"
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(swec.SwecError) as e2:
            ec.Encoder(10, 4, device=0).encode(shards)
        assert e2.value.name in ("SWEC_ERR_NO_DEVICE", "SWEC_ERR_CUDA")
        n = C.c_int(-1)
        assert swec.lib().swec_device_count(C.byref(n)) == -7 and n.value == 0


def test_argument_validation(swec, tmp_path):
    ec = swec.erasure_coding
    enc = ec.Encoder(10, 4, device=-1)
    with pytest.raises(swec.SwecError):
        enc.encode([np.zeros(8, dtype=np.uint8)] * 13)            # wrong shard count
    with pytest.raises(swec.SwecError):
        enc.encode([np.zeros(8, dtype=np.uint8)] * 13 + [np.zeros(9, dtype=np.uint8)])  # ErrShardSize
    with pytest.raises(swec.SwecError):
        enc.reconstruct([None] * 5 + [np.zeros(8, dtype=np.uint8)] * 9)   # ErrTooFewShards
    with pytest.raises(swec.SwecError) as e:
        ec.generate_ec_files(str(tmp_path / "x"), 0, 1 << 30, 1 << 20)    # zero buffer (Fatal in Go)
    assert e.value.name == "SWEC_ERR_INVALID_ARG"
    with pytest.raises(swec.SwecError):
        ec.generate_ec_files(str(tmp_path / "x"), 48, 10000, 100)         # block % buffer != 0
    with pytest.raises(swec.SwecError) as e:
        ec.generate_ec_files(str(tmp_path / "missing"), 50, 10000, 100)   # no .dat
    assert e.value.name == "SWEC_ERR_IO"
    with pytest.raises(swec.SwecError) as e:
        enc.extract_data_shard_device(1, -1, 0, 1)                         # negative .dat size, before any device work
    assert e.value.name == "SWEC_ERR_INVALID_ARG"
    with pytest.raises(swec.SwecError) as e:                              # a shard to rebuild without a buffer, before
        enc.reconstruct_device([None] + [1 << 20] * 13, [0] + [1] * 13, 4096)  # any device work
    assert e.value.name == "SWEC_ERR_INVALID_ARG"


def test_set_option_validation(swec):
    L = swec.lib()
    for name, good, bad in ((b"power_mode", 2, 3), (b"xt_variant", 3, 4), (b"use_aot", 0, 2), (b"stage_slots", 4, 1),
                            (b"enc_threads", 256, 300), (b"jit", 1, 5), (b"host_pieces", 2, 0), (b"host_min_chunk", 65536, 100)):
        assert L.swec_set_option(name, bad) == -1, name
        assert L.swec_set_option(name, good) == 0, name
    assert L.swec_set_option(b"no_such_option", 1) == -1 and L.swec_set_option(None, 1) == -1
    for name, dflt in ((b"power_mode", 1), (b"xt_variant", 0), (b"use_aot", 1), (b"stage_slots", 3), (b"enc_threads", 512),
                       (b"host_pieces", 4), (b"host_min_chunk", 256 << 10)):
        assert L.swec_set_option(name, dflt) == 0


def test_multi_handle_argument_validation(swec):
    """The column-split calls validate the group before touching a device."""
    ec = swec.erasure_coding
    L = swec.lib()
    a, b, c = ec.Encoder(10, 4, device=-1), ec.Encoder(10, 4, device=-1), ec.Encoder(6, 3, device=-1)
    shards = [np.zeros(8192, dtype=np.uint8) for _ in range(14)]
    ptrs = (C.c_void_p * 14)(*[s.ctypes.data for s in shards])
    present = (C.c_uint8 * 14)(*([0] + [1] * 13))

    def group(*encs):
        return (C.c_void_p * len(encs))(*[e._h for e in encs]), len(encs)
    assert L.swec_encode_multi(*group(a, a), ptrs, 8192) == -1            # same handle twice
    assert L.swec_encode_multi(*group(a, c), ptrs, 8192) == -1            # mixed ratios
    assert L.swec_encode_multi(None, 0, ptrs, 8192) == -1
    assert L.swec_encode_multi(*group(a, b), ptrs, 0) == -1               # ErrShardNoData
    assert L.swec_encode_multi(*group(a, b), ptrs, 8192) == -7            # no device: loud, no fallback
    assert b"no CPU fallback" in L.swec_last_error()                      # detail crossed from the worker thread
    assert L.swec_reconstruct_multi(*group(a, b), ptrs, present, 8192, 0) == -7
    few = (C.c_uint8 * 14)(*([0] * 5 + [1] * 9))
    assert L.swec_reconstruct_multi(*group(a, b), ptrs, few, 8192, 0) == -2
    allp = (C.c_uint8 * 14)(*([1] * 14))
    assert L.swec_reconstruct_multi(*group(a, b), ptrs, allp, 8192, 0) == 0   # nothing to do
    out = (C.c_void_p * 14)()
    assert L.swec_alloc_pinned_shards(*group(a, a), 14, 8192, out) == -1      # group checks first
    assert L.swec_alloc_pinned_shards(*group(a, b), 0, 8192, out) == -1
    assert L.swec_alloc_pinned_shards(*group(a, b), 14, 0, out) == -1
    import torch
    if not torch.cuda.is_available():                                       # pinning needs the driver: loud, no leak
        assert L.swec_alloc_pinned_shards(*group(a, b), 14, 8192, out) in (-3, -7)


def test_rebuild_prechecks_need_no_gpu(swec, tmp_path):
    """generateMissingEcFiles bails out before creating outputs when < k shards exist (ec_encoder.go:172-175)."""
    ec = swec.erasure_coding
    base = str(tmp_path / "3")
    for i in range(9):
        open(base + ec.ToExt(i), "wb").write(b"\0" * 16)
    with pytest.raises(swec.SwecError) as e:
        ec.rebuild_ec_files(base)
    assert e.value.name == "SWEC_ERR_TOO_FEW_SHARDS"
    assert sorted(os.listdir(tmp_path)) == ["3.ec%02d" % i for i in range(9)]
    # all shards present: nothing to do, no device touched
    for i in range(9, 14):
        open(base + ec.ToExt(i), "wb").write(b"\0" * 16)
    assert ec.rebuild_ec_files(base) == []


def test_write_dat_file_roundtrip(swec, oracle, tmp_path):
    """WriteDatFile over every shape of the last row, with k = 10, large = 10,000 and small = 100."""
    ec = swec.erasure_coding
    rng = np.random.default_rng(9)
    for dat_size in (
        300_000,        # 3 whole large rows (k * large = 100,000)
        307_000,        # large rows + 7 full small rows, no tail
        307_037,        # a tail shorter than one small block
        1_234_567,      # a tail of 567 bytes: it ends inside shard 5
        307_999,        # a tail of k * small - 1 bytes
    ):
        d = tmp_path / str(dat_size)
        d.mkdir()
        dat = rng.integers(0, 256, dat_size, dtype=np.uint8)
        shards = oracle.encode_dat_image(dat, buffer_size=50, large=10000, small=100)
        names = []
        for i in range(10):
            names.append(str(d / ("5.ec%02d" % i)))
            shards[i].tofile(names[-1])
        ec.write_dat_file(str(d / "out"), len(dat), names, 10, 10000, 100)
        assert (np.fromfile(str(d / "out.dat"), dtype=np.uint8) == dat).all(), dat_size


def test_jit_source_compiles_for_sm90a_without_gpu(swec):
    """The run-time specialised kernel source (prelude + generated combiner) goes through NVRTC for
    sm_90a without a GPU: catches generator / prelude errors before any GPU time is spent."""
    import time
    from oracle import rs_numpy as rn
    L = swec.lib()
    cases = [rn.fused_reconstruct_rows(10, 4, [i not in e for i in range(14)])[2]
             for e in ((0, 1, 2, 3), (5,), (2, 11), (10, 11, 12, 13))]
    cases.append(rn.build_matrix(6, 9)[6:])
    cases.append(rn.build_matrix(20, 28)[20:])          # 8 output rows: the per-launch maximum
    for rows in cases:
        rows = np.ascontiguousarray(rows, dtype=np.uint8)
        size, steps, xors = C.c_size_t(0), C.c_int(0), C.c_int(0)
        t0 = time.perf_counter()
        rc = L.swec_debug_jit_compile(rows.shape[0], rows.shape[1], rows.ctypes.data, C.byref(size),
                                      C.byref(steps), C.byref(xors))
        if rc == -8 and b"not available" in L.swec_last_error():
            pytest.skip("NVRTC not installed here")
        assert rc == 0, L.swec_last_error()
        assert size.value > 1000 and steps.value <= 7 * rows.shape[0]
        print(rows.shape, size.value, steps.value, xors.value, round(time.perf_counter() - t0, 3))
    # the opt-in formulation with shared power chains compiles too, with fewer steps for the worst-case decode matrix
    assert L.swec_set_option(b"jit_share_powers", 1) == 0
    try:
        rows = np.ascontiguousarray(cases[0], dtype=np.uint8)
        size, steps, xors = C.c_size_t(0), C.c_int(0), C.c_int(0)
        assert L.swec_debug_jit_compile(4, 10, rows.ctypes.data, C.byref(size), C.byref(steps), C.byref(xors)) == 0
        assert size.value > 1000 and steps.value == 21
    finally:
        assert L.swec_set_option(b"jit_share_powers", 0) == 0


def test_device_spread_order_without_devices(swec):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    order, cnt = (C.c_int * 8)(), C.c_int(-1)
    assert swec.lib().swec_device_spread_order(order, 8, C.byref(cnt)) == -7 and cnt.value == 0     # SWEC_ERR_NO_DEVICE
    assert swec.lib().swec_device_spread_order(None, 8, C.byref(cnt)) == -1


def test_cubin_disk_cache_and_aot_table(swec, tmp_path, monkeypatch):
    """The decode-kernel cache outlives the process: a matrix compiled once is loaded from the on-disk cubin cache
    the next time (no NVRTC compile), and the 15 most common reconstruct matrices are compiled with the library."""
    import time
    from oracle import rs_numpy as rn
    L = swec.lib()
    aot = C.c_int(0)
    assert L.swec_jit_stats(None, None, C.byref(aot), None) == 0 and aot.value == 15       # 14 single losses + shards 0-3
    monkeypatch.setenv("SWEC_CACHE_DIR", str(tmp_path / "cubins"))
    rows = np.ascontiguousarray(rn.fused_reconstruct_rows(10, 4, [i not in (3, 7, 12) for i in range(14)])[2], dtype=np.uint8)

    def compile_once():
        c0, h0 = C.c_uint64(0), C.c_uint64(0)
        L.swec_jit_stats(C.byref(c0), C.byref(h0), None, None)
        size = C.c_size_t(0)
        t0 = time.perf_counter()
        rc = L.swec_debug_jit_compile(rows.shape[0], rows.shape[1], rows.ctypes.data, C.byref(size), None, None)
        dt = time.perf_counter() - t0
        c1, h1 = C.c_uint64(0), C.c_uint64(0)
        L.swec_jit_stats(C.byref(c1), C.byref(h1), None, None)
        return rc, size.value, c1.value - c0.value, h1.value - h0.value, dt

    rc, size, compiles, hits, _ = compile_once()
    if rc == -8 and b"not available" in L.swec_last_error():
        pytest.skip("NVRTC not installed here")
    assert rc == 0 and (compiles, hits) == (1, 0)
    files = list((tmp_path / "cubins").glob("*.cubin"))
    assert len(files) == 1 and files[0].stat().st_size == size
    rc, size2, compiles, hits, dt = compile_once()
    assert rc == 0 and (compiles, hits) == (0, 1) and size2 == size and dt < 0.1, dt
    # a cache directory that others can write to is not trusted with executable code: the cache is off, NVRTC compiles
    os.chmod(tmp_path / "cubins", 0o777)
    rc, _, compiles, hits, _ = compile_once()
    assert rc == 0 and (compiles, hits) == (1, 0)
    os.chmod(tmp_path / "cubins", 0o700)
    rc, _, compiles, hits, _ = compile_once()
    assert rc == 0 and (compiles, hits) == (0, 1)
    monkeypatch.setenv("SWEC_NO_DISK_CACHE", "1")
    rc, _, compiles, hits, _ = compile_once()
    assert rc == 0 and (compiles, hits) == (1, 0)


def test_layout_arithmetic_fuzz_against_oracle(swec, oracle):
    """LocateData / ToShardIdAndOffset / expected shard size for random block sizes, ratios, volume sizes and reads:
    libswec against the oracle's restatement of ec_locate.go:16-98 and disk_location_ec.go:428-448 (hypothesis)."""
    from hypothesis import HealthCheck, given, settings
    from hypothesis import strategies as st
    from oracle import rs_numpy as rn
    ec = swec.erasure_coding

    @settings(max_examples=300, deadline=None, derandomize=True, suppress_health_check=list(HealthCheck))
    @given(k=st.integers(1, 20), small=st.integers(1, 300), mult=st.integers(1, 50), rows=st.integers(0, 4),
           extra=st.integers(0, 20000), off_frac=st.floats(0, 1), size=st.integers(1, 5000))
    def check(k, small, mult, rows, extra, off_frac, size):
        large = small * mult
        dat_size = rows * large * k + extra
        sizes = (ec.expected_shard_size(dat_size, k, large, small), oracle.expected_shard_size(dat_size, k, large, small),
                 rn.expected_shard_size(dat_size, k, large, small))
        assert sizes[0] == sizes[1] == sizes[2], sizes
        if dat_size == 0:
            return
        offset = int(off_frac * (dat_size - 1))
        size = min(size, dat_size - offset)
        shard_dat_size = dat_size // k
        got = ec.locate_data(large, small, shard_dat_size, offset, size, k)
        want = rn.locate_data(large, small, shard_dat_size, offset, size, k)
        assert [tuple(g) for g in got] == [tuple(w) for w in want], (k, large, small, dat_size, offset, size)
        assert sum(g[2] for g in got) == size
        for iv in got:
            assert ec.interval_to_shard(iv, large, small, k) == rn.interval_to_shard(iv, large, small, k)

    check()


def _split_top_level(args: str) -> list[str]:
    out, depth, cur = [], 0, ""
    for ch in args:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == "," and depth == 0:
            out.append(cur)
            cur = ""
        else:
            cur += ch
    return [a for a in out + [cur] if a.strip()]


def test_cgo_shim_calls_match_the_header():
    """Go is not installed here, so the shim (integration/go/ec_swec.go, also quoted in INTEGRATION.md) cannot be
    compiled; at least every C.swec_* call in it must name a function include/swec.h declares, with the declared
    number of arguments, and every C.SWEC_* constant must exist."""
    header = open(os.path.join(ROOT, "include", "swec.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    decls = {}
    for m in re.finditer(r"\b(swec_\w+)\s*\(([^;{]*?)\)\s*;", header, flags=re.S):
        params = m.group(2).strip()
        decls[m.group(1)] = 0 if params in ("", "void") else len(_split_top_level(params))
    go = open(os.path.join(ROOT, "integration", "go", "ec_swec.go")).read()
    calls = 0
    for m in re.finditer(r"C\.(swec_\w+)\(", go):
        name = m.group(1)
        if name in ("swec_encoder", "swec_ec_volume", "swec_needle_read"):      # type names used in conversions
            continue
        assert name in decls, f"{name} is not declared in swec.h"
        depth, i = 1, m.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(go[i], 0)
            i += 1
        args = _split_top_level(go[m.end():i - 1])
        assert len(args) == decls[name], f"{name}: shim passes {len(args)} arguments, header declares {decls[name]}"
        calls += 1
    assert calls >= 15
    for const in set(re.findall(r"C\.(SWEC_\w+)", go)):
        assert re.search(rf"\b{const}\b", header), const
    md = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    block = re.search(r"```go\n(//go:build swec && cgo.*?)```", md, re.S).group(1)
    assert block.strip() in go, "INTEGRATION.md's listing and integration/go/ec_swec.go have drifted apart"
