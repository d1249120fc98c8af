"""seaweedfs_b200/build.py — builds libswec.so (the C-ABI library, include/swec.h) in-tree.

Steps:
  1. host tool `swec_codegen` (codegen.cc) emits the straight-line RS(10,4) encode combiner;
  2. the JIT prelude (apply_params.h + device_common.cuh) is embedded as a string literal;
  3. nvcc compiles everything for sm_90a only (-gencode arch=compute_90a,code=sm_90a -lineinfo)
     into seaweedfs_b200/libswec.so with cudart linked statically (no libcuda/NVRTC link-time
     dependency: the library must load on a machine without a GPU).
nvcc cross-compiles without a GPU, so this runs in the CPU-only build container.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
GEN = os.path.join(CSRC, "generated")
LIB = os.path.join(HERE, "libswec.so")
ROOT = os.path.dirname(HERE)

SOURCES = ["kernels.cu", "aot_recon.cu", "needles.cu", "damage.cu", "needle_damage.cu", "sketch.cu", "engine.cc", "host_seam.cc", "ec_files.cc", "ec_index.cc", "ec_volume.cc", "volume_format.cc", "staging.cc",
           "jit.cc", "codegen.cc", "gf256.cc"]
HEADERS = ["apply_params.h", "device_common.cuh", "tma_fetch.cuh", "kernels.h", "engine.h", "host_seam.h", "gf256.h", "codegen.h", "io_pool.h", "mini_json.h",
           "volume_format.h", "needle_format.h", "needles.h", "damage.h", "needle_damage.h", "sketch.h", "locate_decode.cuh", "stripe_map.h", "staging.h", os.path.join(ROOT, "include", "swec.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function", "-cudart", "static"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found — libswec.so cannot be built (there is no CPU fallback)")


def _run(cmd: list[str], **kw) -> None:
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, **kw)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("command failed: " + " ".join(cmd))


def _stamp() -> str:
    h = hashlib.sha256()
    paths = [os.path.join(CSRC, s) for s in SOURCES + ["codegen_main.cc"]] + \
            [p if os.path.isabs(p) else os.path.join(CSRC, p) for p in HEADERS] + [os.path.abspath(__file__)]
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(os.environ.get("SWEC_EXTRA_NVCC_FLAGS", "").encode())
    h.update(os.environ.get("SWEC_CODEGEN_FLAGS", "").encode())
    return h.hexdigest()


def generate() -> None:
    os.makedirs(GEN, exist_ok=True)
    tool = os.path.join(GEN, "swec_codegen")
    _run(["g++", "-O2", "-std=c++17", "-o", tool] +
         [os.path.join(CSRC, s) for s in ("codegen_main.cc", "codegen.cc", "gf256.cc")])
    # SWEC_CODEGEN_FLAGS="--share-powers --search-basis" builds the kernels with the CPU-verified but not yet measured
    # formulation of DESIGN.md §9.4 (default: none — the shipped kernels are the ones the test suite and bench.py run)
    gen_flags = os.environ.get("SWEC_CODEGEN_FLAGS", "").split()
    out = subprocess.run([tool, "--rs", "10", "4", "--name", "Rs10x4Encode"] + gen_flags, check=True,
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout
    with open(os.path.join(GEN, "gen_rs10x4_encode.inc"), "w") as f:
        f.write(out)
    # the same combiner under a second name: kernels.cu binds it to the low-power multiply-by-2 step
    with open(os.path.join(GEN, "gen_rs10x4_encode_lp.inc"), "w") as f:
        f.write(out.replace("struct Rs10x4Encode ", "struct Rs10x4EncodeLP "))
    # reconstruct matrices compiled ahead of time (aot_recon.cu): combiners + the matrix table they are found by
    for emit, name in (("structs", "gen_aot_recon.inc"), ("keys", "gen_aot_recon_keys.inc")):
        text = subprocess.run([tool, "--aot-recon", "10", "4", "--emit", emit] +
                              [f for f in gen_flags if f == "--share-powers"], check=True,
                              stdout=subprocess.PIPE, text=True).stdout
        with open(os.path.join(GEN, name), "w") as f:
            f.write(text)
    # JIT prelude: the two device headers, flattened (NVRTC cannot #include from disk)
    text = []
    for name in ("apply_params.h", "device_common.cuh"):
        with open(os.path.join(CSRC, name)) as f:
            for line in f:
                if line.startswith("#pragma once") or line.startswith('#include "apply_params.h"'):
                    continue
                text.append(line)
    with open(os.path.join(GEN, "device_common_src.inc"), "w") as f:
        f.write('R"SWECSRC(' + "".join(text) + ')SWECSRC"\n')


def build(force: bool = False, verbose: bool = False) -> str:
    stamp_path = os.path.join(GEN, "build.stamp")
    stamp = _stamp()
    if not force and os.path.exists(LIB) and os.path.exists(stamp_path):
        with open(stamp_path) as f:
            if f.read().strip() == stamp:
                return LIB
    generate()
    extra = os.environ.get("SWEC_EXTRA_NVCC_FLAGS", "").split()
    # one nvcc -c per source, in parallel (the two kernel files dominate), then one link step
    from concurrent.futures import ThreadPoolExecutor
    objdir = os.path.join(GEN, "obj")
    os.makedirs(objdir, exist_ok=True)
    common = [_nvcc()] + NVCC_FLAGS + extra + ["-I", CSRC, "-I", GEN]
    objs = [os.path.join(objdir, os.path.splitext(src)[0] + ".o") for src in SOURCES]

    def compile_one(pair):
        src, obj = pair
        cmd = common + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd))
        _run(cmd)
    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 2)) as ex:
        list(ex.map(compile_one, zip(SOURCES, objs)))
    cmd = common + ["-shared", "-o", LIB] + objs + ["-ldl", "-lpthread"]
    if verbose:
        print(" ".join(cmd))
    _run(cmd)
    with open(stamp_path, "w") as f:
        f.write(stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
