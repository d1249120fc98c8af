"""Cost of naming the needles that located damage hits (swec_ec_volume_locate_needle_damage) over the plain locate
(swec_locate_ec_damage) on the same shard files: 14 shard files of --gib GiB each (default 1), from the page cache, with
an .ecx of records of 4-200 KiB tiling the volume.  Two sets: clean, and one flipped byte per MiB of data shard 3.
The calls alternate, --reps times each.  What the needle call adds is pass 2 (the flagged pages read again, corrected on
a copy, re-encoded) and the join; on a clean set it adds nothing.  One JSON line to stdout (and --out).

    python scripts/bench_needle_damage.py [--gib 1] [--reps 3] [--out FILE]
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

SEED = 0x4EEDBE
MIB = 1 << 20


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()

    import torch

    import seaweedfs_b200
    from oracle import rs_numpy as rn
    from seaweedfs_b200 import erasure_coding as ec

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    L = seaweedfs_b200.lib()
    n = int(a.gib * (1 << 30)) // MIB * MIB
    res = {"gpu": gpu, "shard_bytes": n}
    tmp = tempfile.mkdtemp(prefix="swec_needle_damage_")
    try:
        if shutil.disk_usage(tmp).free < 2 * 14 * n:
            res["check"] = "not measured: too little free disk"
            print(json.dumps(res))
            return
        base = os.path.join(tmp, "1")
        shards = [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(14)]
        for i in range(10):
            seaweedfs_b200._native.check(L.swec_synth_fill_device(0, shards[i].data_ptr(), i * n, n, SEED, None))
        enc = ec.Encoder(10, 4, device=0)
        enc.encode_device([s.data_ptr() for s in shards[:10]], [s.data_ptr() for s in shards[10:]], n)
        enc.synchronize()
        for i, s in enumerate(shards):
            s.cpu().numpy().tofile(base + ".ec%02d" % i)
        del shards
        torch.cuda.empty_cache()
        dat_size = 10 * n                      # below 10 GiB: small rows only, as LocateData sees them
        rng = np.random.default_rng(SEED)
        sizes = rng.integers(4096, 200 * 1024, dat_size // 4096)
        ends = 8 + np.cumsum((sizes + 16 + 4 + 8 + 8) // 8 * 8)
        offs = np.concatenate([[8], ends[:-1]])
        keep = ends <= dat_size
        entries = [rn._entry(j + 1, int(o) // 8, int(s)) for j, (o, s) in enumerate(zip(offs[keep], sizes[keep]))]
        open(base + ".ecx", "wb").write(b"".join(entries))
        json.dump({"version": 3, "datFileSize": str(dat_size), "ecShardConfig": {"dataShards": 10, "parityShards": 4}},
                  open(base + ".vif", "w"))
        res["records"] = len(entries)
        vol = ec.EcVolume(base)
        ok = True

        def alternate(tag):
            loc, nd = [], []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                plain = ec.locate_ec_damage(base)
                t1 = time.perf_counter()
                got = vol.locate_needle_damage(max_needles=1 << 20)
                t2 = time.perf_counter()
                loc.append(t1 - t0)
                nd.append(t2 - t1)
            res.update({f"{tag}_locate_s": loc, f"{tag}_needle_damage_s": nd,
                        f"{tag}_ratio_best": min(nd) / min(loc), f"{tag}_ratio_median": float(np.median(nd) / np.median(loc))})
            return plain, got

        plain, got = alternate("clean")
        ok = ok and plain["ok"] and got["ok"] and got["n_needles"] == 0
        with open(base + ".ec03", "r+b") as f:          # one flipped byte per MiB of data shard 3
            for o in range(12345, n, MIB):
                f.seek(o)
                b = f.read(1)[0]
                f.seek(o)
                f.write(bytes([b ^ 0x40]))
        plain, got = alternate("one_byte_per_MiB")
        flips = len(range(12345, n, MIB))
        ok = ok and plain["shards"] == {3: (flips, 12345, 12345 + (flips - 1) * MIB)}
        ok = ok and sum(r["damaged_bytes"] for r in got["needles"]) + got["unowned"][0] == flips
        res["needles_named"] = got["n_needles"]
        vol.close()
        res["check"] = "ok" if ok else "MISMATCH"
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
