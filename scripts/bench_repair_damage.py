"""Rate of in-place repair (swec_correct_damage_device, swec_repair_ec_damage) against what it replaces.

- Device level, 14 shards of 3 GiB in HBM (a 30 GiB volume's): a clean correcting pass alternated with a locate pass in
  the same process (they should cost the same), then 1 % of the columns damaged in one shard, damaged again between
  repetitions outside the timed region.
- File level, where the disk has room: the first --file-gib of every shard as shard files, a few MiB of damage in one
  data shard, repair_ec_damage against deleting that shard and running rebuild_ec_files, alternating.  Both read the
  other shards from the page cache, and both timings include making the written bytes durable (the repair's own
  fdatasync; an fdatasync of the rebuilt file); the page cache holds nothing dirty when a timed call starts.  Bytes
  written are reported beside the seconds.

One JSON line to stdout (and --out), with the GPU's name, power limit and max SM clock.

    python scripts/bench_repair_damage.py [--gib 3] [--reps 10] [--file-gib 1] [--damage-mib 4] [--out FILE]
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

SEED = 0xDA3A6E


def timed(fn, reps, before=None):
    """best and median seconds of fn(); before() runs untimed ahead of every repetition"""
    out = []
    for _ in range(reps):
        if before:
            before()
        t0 = time.perf_counter()
        fn()
        out.append(time.perf_counter() - t0)
    return min(out), float(np.median(out))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--file-gib", type=float, default=1)
    ap.add_argument("--damage-mib", type=float, default=4)
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
    ok = enc.correct_damage_device(ptrs, n)["damaged_columns"] == 0      # warm-up of both, and the set must be clean
    ok = ok and enc.locate_damage_device(ptrs, n)["damaged_columns"] == 0
    res = {"gpu": gpu, "shard_bytes": n}
    for _ in range(2):                                                    # alternate: locate, correct, locate, correct
        l_best, l_med = timed(lambda: enc.locate_damage_device(ptrs, n), a.reps)
        c_best, c_med = timed(lambda: enc.correct_damage_device(ptrs, n), a.reps)
    res.update({"locate_clean_s_best": l_best, "locate_clean_s_median": l_med,
                "correct_clean_s_best": c_best, "correct_clean_s_median": c_med})

    # 1 % of the columns damaged in one data shard, spread evenly; damaged again before every repetition
    def spoil():
        shards[3][::100] ^= 1
        torch.cuda.synchronize()

    spoil()
    rep = enc.locate_damage_device(ptrs, n)
    ok = ok and rep["shards"].get(3, (0,))[0] == (n + 99) // 100 and rep["uncorrectable_columns"] == 0
    l_best, l_med = timed(lambda: enc.locate_damage_device(ptrs, n), 3)
    rep = enc.correct_damage_device(ptrs, n)
    ok = ok and rep["shards"].get(3, (0,))[0] == (n + 99) // 100
    ok = ok and enc.locate_damage_device(ptrs, n)["damaged_columns"] == 0
    c_best, c_med = timed(lambda: enc.correct_damage_device(ptrs, n), a.reps, before=spoil)
    ok = ok and enc.locate_damage_device(ptrs, n)["damaged_columns"] == 0
    res.update({"one_percent_locate_s_best": l_best, "one_percent_locate_s_median": l_med,
                "one_percent_correct_s_best": c_best, "one_percent_correct_s_median": c_med})

    # file level: repair in place against delete-and-rebuild of the damaged shard
    fsz = min(n, int(a.file_gib * (1 << 30)) & ~4095)
    dmg = min(fsz, int(a.damage_mib * (1 << 20)))
    tmp = tempfile.mkdtemp(prefix="swec_repair_")
    try:
        if shutil.disk_usage(tmp).free > 3 * 14 * fsz:
            base = os.path.join(tmp, "1")
            for i, s in enumerate(shards):
                s[:fsz].cpu().numpy().tofile(base + ".ec%02d" % i)
            del shards
            torch.cuda.empty_cache()
            path = base + ".ec03"
            at = fsz // 3
            with open(path, "rb") as f:
                f.seek(at)
                good = np.frombuffer(f.read(dmg), dtype=np.uint8)

            def spoil_file():  # and nothing left dirty in the page cache for the timed call to flush
                with open(path, "r+b") as f:
                    f.seek(at)
                    f.write((good ^ 0x5A).tobytes())
                os.sync()

            ok = ok and ec.repair_ec_damage(base)["damaged_columns"] == 0
            spoil_file()
            written = {}

            def repair():
                r = ec.repair_ec_damage(base)
                written["repair"] = sum(length for sid, _, length in r["ranges"] if sid >= 0)
                assert r["ok"] and set(r["shards"]) == {3}

            def rebuild():  # made durable, as the repair's writes are
                os.remove(path)
                assert ec.rebuild_ec_files(base) == [3]
                fd = os.open(path, os.O_RDONLY)
                os.fdatasync(fd)
                os.close(fd)
                written["rebuild"] = os.path.getsize(path)

            rp, rb = [], []
            for _ in range(3):
                rp.append(timed(repair, 1, before=spoil_file)[0])
                rb.append(timed(rebuild, 1, before=spoil_file)[0])
            ok = ok and ec.locate_ec_damage(base)["ok"]
            res.update({"file_shard_bytes": fsz, "file_damage_bytes": dmg, "file_repair_s": rp, "file_rebuild_s": rb,
                        "file_repair_bytes_written": written["repair"], "file_rebuild_bytes_written": written["rebuild"]})
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
