"""Cost of the checked rebuild (swec_reconstruct_checked_device, swec_rebuild_ec_files_checked) against plain rebuild.

- Device level, 14 shards of 3 GiB in HBM (a 30 GiB volume's) with shard 0 lost: swec_reconstruct_device and
  swec_reconstruct_checked_device alternated, best and median of --reps each, on a clean set and again with 1 % of the
  columns damaged in one present data shard.  The checked call never writes present shards, so the damage stays put
  between repetitions.  Both fused matrices are warmed (run-time specialisation included) before timing.  Algorithmic
  bytes per column: 11 for plain (10 read, 1 written), 20 for checked (10 read and 4 written by the apply, 3 computed
  and 3 stored check bytes read by the locator); the rate is given as a fraction of 3.35 TB/s.
- File level, where the disk has room: the first --file-gib of every shard as shard files in the page cache, shard 0
  lost, rebuild_ec_files and rebuild_ec_files_checked alternated over three calls each.  Bytes read and written are the
  process's rchar / wchar deltas over the call (/proc/self/io) where the kernel exposes them, else counted from the
  shard files each call reads and writes (and marked so).

One JSON line to stdout (and --out), with the GPU's name, power limit and max SM clock.

    python scripts/bench_checked_rebuild.py [--gib 3] [--reps 10] [--file-gib 1] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED = 0xC4EC
HBM_PEAK = 3.35e12


def io_counts():
    """(rchar, wchar) of the process, or None where /proc/self/io is not readable"""
    try:
        with open("/proc/self/io") as f:
            d = dict(line.split(": ") for line in f.read().splitlines() if ": " in line)
        return int(d["rchar"]), int(d["wchar"])
    except (OSError, KeyError, ValueError):
        return None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--file-gib", type=float, default=1)
    ap.add_argument("--out")
    a = ap.parse_args()

    import torch

    import seaweedfs_b200
    from seaweedfs_b200 import erasure_coding as ec

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    L = seaweedfs_b200.lib()
    n = int(a.gib * (1 << 30)) & ~4095
    shards = [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(14)]
    for i in range(10):
        seaweedfs_b200._native.check(L.swec_synth_fill_device(0, shards[i].data_ptr(), i * n, n, SEED, None))
    enc = ec.Encoder(10, 4, device=0)
    enc.encode_device([s.data_ptr() for s in shards[:10]], [s.data_ptr() for s in shards[10:]], n)
    enc.synchronize()
    ptrs = [s.data_ptr() for s in shards]
    present = [0] + [1] * 13
    want0 = shards[0].clone()

    def plain():
        enc.reconstruct_device(ptrs, present, n)
        enc.synchronize()

    def checked():
        return enc.reconstruct_checked_device(ptrs, present, n)

    ok = True
    for _ in range(2):                                                    # warm-up, specialised kernels included
        plain()
        ok = ok and checked()["damaged_columns"] == 0
    ok = ok and bool(torch.equal(shards[0], want0))
    res = {"gpu": gpu, "shard_bytes": n}

    def alternate(tag):
        tp, tc = [], []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            plain()
            tp.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            checked()
            tc.append(time.perf_counter() - t0)
        for name, t, per_col in (("plain", tp, 11), ("checked", tc, 20)):
            best = min(t)
            res[f"{tag}_{name}_s_best"] = best
            res[f"{tag}_{name}_s_median"] = float(np.median(t))
            res[f"{tag}_{name}_frac_of_3.35TBps"] = per_col * n / best / HBM_PEAK

    alternate("clean")
    shards[3][::100] ^= 1                                               # 1 % of the columns of a present data shard
    torch.cuda.synchronize()
    rep = checked()
    ok = ok and rep["shards"].get(3, (0,))[0] == (n + 99) // 100 and rep["uncorrectable_columns"] == 0
    ok = ok and bool(torch.equal(shards[0], want0))
    alternate("one_percent")
    ok = ok and bool(torch.equal(shards[0], want0))
    shards[3][::100] ^= 1
    torch.cuda.synchronize()
    res["bytes_per_column"] = {"plain": 11, "checked": 20}

    # file level: plain against checked rebuild of shard 0, the other shards in the page cache
    fsz = min(n, int(a.file_gib * (1 << 30)) & ~((1 << 20) - 1))
    tmp = tempfile.mkdtemp(prefix="swec_checked_")
    try:
        if shutil.disk_usage(tmp).free > 3 * 14 * fsz:
            base = os.path.join(tmp, "1")
            for i, s in enumerate(shards):
                s[:fsz].cpu().numpy().tofile(base + ".ec%02d" % i)
            del shards
            torch.cuda.empty_cache()
            path = base + ".ec00"
            good = np.fromfile(path, dtype=np.uint8)
            counts = {}

            def run(name, call):
                os.remove(path)
                c0 = io_counts()
                t0 = time.perf_counter()
                out = call(base)
                dt = time.perf_counter() - t0
                c1 = io_counts()
                if c0 and c1:
                    counts[name] = (c1[0] - c0[0], c1[1] - c0[1], "rchar/wchar")
                else:                       # plain reads the first 10 present shards, checked all 13; both write 1
                    counts[name] = ((10 if name == "plain" else 13) * fsz, fsz, "counted from the shards read")
                return dt, out

            tp, tc = [], []
            run("plain", ec.rebuild_ec_files)                             # warm-up of both
            run("checked", ec.rebuild_ec_files_checked)
            for _ in range(3):
                dt, _ = run("plain", ec.rebuild_ec_files)
                tp.append(dt)
                dt, rep = run("checked", ec.rebuild_ec_files_checked)
                tc.append(dt)
                ok = ok and rep["ok"] and rep["damaged_columns"] == 0
            ok = ok and bool((np.fromfile(path, dtype=np.uint8) == good).all())
            res.update({"file_shard_bytes": fsz, "file_plain_s": tp, "file_checked_s": tc,
                        "file_plain_bytes_read": counts["plain"][0], "file_plain_bytes_written": counts["plain"][1],
                        "file_checked_bytes_read": counts["checked"][0],
                        "file_checked_bytes_written": counts["checked"][1], "file_bytes_source": counts["checked"][2]})
        else:
            res["file_level"] = "not measured: too little free disk"
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    res["check"] = "ok" if ok else "MISMATCH"
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
