"""Rate of the damage locator (swec_locate_damage_device) over the 14 shards of a 30 GiB volume in HBM (3 GiB each),
against swec_encode_device on the same data in the same process; its slow path; and, where the disk has room, the
file-level swec_locate_ec_damage against swec_verify_ec_files on the same shard files, alternating.

Algorithmic bytes of a clean pass are 22 per column for RS(10,4): read 10 data bytes, write and read 4 computed parity
bytes, read 4 stored parity bytes.  One JSON line to stdout (and --out).

    python scripts/bench_locate_damage.py [--gib 3] [--reps 10] [--file-gib 1] [--out FILE]
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

HBM_PEAK = 3.35e12  # H100 SXM data sheet
SEED = 0xDA3A6E


def timed(fn, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append(time.perf_counter() - t0)
    return min(out), float(np.median(out))


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
    data, parity = [s.data_ptr() for s in shards[:10]], [s.data_ptr() for s in shards[10:]]
    ptrs = data + parity

    def encode():
        enc.encode_device(data, parity, n)
        enc.synchronize()

    encode()
    rep = enc.locate_damage_device(ptrs, n)                 # warm-up, and the clean pass must be clean
    ok = rep["damaged_columns"] == 0
    res = {"gpu": gpu, "shard_bytes": n}
    for _ in range(2):                                       # alternate: encode, locate, encode, locate
        e_best, e_med = timed(encode, a.reps)
        l_best, l_med = timed(lambda: enc.locate_damage_device(ptrs, n), a.reps)
    algo = 22 * n
    res.update({"locate_clean_s_best": l_best, "locate_clean_s_median": l_med,
                "locate_GBps_best": algo / l_best / 1e9, "locate_GBps_median": algo / l_med / 1e9,
                "locate_fraction_of_3.35TBps_best": algo / l_best / HBM_PEAK,
                "encode_s_best": e_best, "encode_s_median": e_med,
                "encode_GBps_best": 14 * n / e_best / 1e9})

    # slow path 1: 1 % of the columns damaged in one data shard, spread evenly (every warp decodes some)
    shards[3][::100] ^= 1
    torch.cuda.synchronize()
    rep = enc.locate_damage_device(ptrs, n)
    ok = ok and rep["shards"].get(3, (0,))[0] == (n + 99) // 100 and rep["uncorrectable_columns"] == 0
    best, med = timed(lambda: enc.locate_damage_device(ptrs, n), 3)
    res.update({"one_percent_in_one_shard_s_best": best, "one_percent_in_one_shard_s_median": med})
    shards[3][::100] ^= 1
    # slow path 2: two data shards damaged over the same 1 GiB, radius 2 (the longest search: a data pair)
    g = min(n, 1 << 30)
    shards[2][:g] ^= 0x33
    shards[6][:g] ^= 0x05
    torch.cuda.synchronize()
    rep = enc.locate_damage_device(ptrs, n, radius=2)
    ok = ok and rep["shards"] == {2: (g, 0, g - 1), 6: (g, 0, g - 1)}
    best, med = timed(lambda: enc.locate_damage_device(ptrs, n, radius=2), 3)
    res.update({"two_shards_1GiB_radius2_s_best": best, "two_shards_1GiB_radius2_s_median": med})
    shards[2][:g] ^= 0x33
    shards[6][:g] ^= 0x05
    torch.cuda.synchronize()

    # file level, if the disk has room: the first --file-gib of every shard as shard files
    fsz = min(n, int(a.file_gib * (1 << 30)) & ~4095)
    tmp = tempfile.mkdtemp(prefix="swec_locate_")
    try:
        if shutil.disk_usage(tmp).free > 3 * 14 * fsz:
            base = os.path.join(tmp, "1")
            for i, s in enumerate(shards):
                s[:fsz].cpu().numpy().tofile(base + ".ec%02d" % i)
            del shards
            torch.cuda.empty_cache()
            ok = ok and ec.locate_ec_damage(base)["ok"] and ec.verify_ec_files(base)[0]
            v, lo = [], []
            for _ in range(3):
                v.append(timed(lambda: ec.verify_ec_files(base), 1)[0])
                lo.append(timed(lambda: ec.locate_ec_damage(base), 1)[0])
            res.update({"file_shard_bytes": fsz, "file_verify_s": v, "file_locate_s": lo,
                        "file_verify_GBps_best": 14 * fsz / min(v) / 1e9, "file_locate_GBps_best": 14 * fsz / min(lo) / 1e9})
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
