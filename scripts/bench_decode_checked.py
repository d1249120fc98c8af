"""Cost of the checked decode (swec_ec_shards_to_volume_checked, swec_decode_data_checked_device) against plain decode.

- Volume level: a synthetic EC volume of --gib GiB (random needle bytes, 64 MiB needles, encoded by
  swec_ec_shards_generate) in a temporary directory, its shards in the page cache.  swec_ec_shards_to_volume (every data
  shard present, the only input it takes) and swec_ec_shards_to_volume_checked are alternated, --file-reps calls each,
  on three sets: clean with all 14 shards; shards 3 and 12 lost; all 14 shards with one flipped byte every MiB of data
  shard 5.  The decoded .dat is checked against the original after the timed calls (checked: every set; plain: the
  clean one).  The plain call reads the 10 data shards and copies them with copy_file_range; the checked call reads the
  (k + c) present shards and pays PCIe both ways.
- Device level: 14 shards of --dev-gib GiB in HBM with shard 0 lost, swec_reconstruct_device(data_only=1) and
  swec_decode_data_checked_device alternated, best and median of --reps each.

One JSON line to stdout and to --out (default profiles/bench_decode_checked.json), with the GPU's name, power limit and
max SM clock.

    python scripts/bench_decode_checked.py [--gib 1] [--file-reps 3] [--dev-gib 3] [--reps 10] [--out FILE]
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED = 0xDEC0
NEEDLE = 64 << 20          # bytes per needle record: header 16 + data + checksum 4 + timestamp 8 + padding 8


def lay_down_volume(base: str, gib: float) -> tuple[int, str]:
    """<base>.dat/.idx of a version-3 volume of 64 MiB needles, encoded by swec_ec_shards_generate; the .dat and .idx
    are removed afterwards.  Returns (dat size, sha256 of the .dat)."""
    from seaweedfs_b200 import erasure_coding as ec
    n = max(1, int(gib * (1 << 30)) // NEEDLE)
    rng = np.random.default_rng(SEED)
    digest = hashlib.sha256()
    with open(base + ".dat", "wb") as f:
        head = bytes([3, 0, 0, 0, 0, 0, 0, 0])
        f.write(head)
        digest.update(head)
        for _ in range(n):
            b = rng.bytes(NEEDLE)
            f.write(b)
            digest.update(b)
    with open(base + ".idx", "wb") as f:
        for i in range(n):
            f.write(struct.pack(">QII", i + 1, (8 + i * NEEDLE) // 8, NEEDLE - 36))
    ec.volume_ec_shards_generate(base)
    os.remove(base + ".dat")
    os.remove(base + ".idx")
    return 8 + n * NEEDLE, digest.hexdigest()


def file_digest(path: str) -> str:
    h = hashlib.sha256()
    with open(path, "rb") as f:
        while b := f.read(64 << 20):
            h.update(b)
    return h.hexdigest()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1)
    ap.add_argument("--file-reps", type=int, default=3)
    ap.add_argument("--dev-gib", type=float, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "bench_decode_checked.json"))
    a = ap.parse_args()

    import torch

    import seaweedfs_b200
    from seaweedfs_b200 import erasure_coding as ec

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    res = {"gpu": gpu}
    ok = True

    # ---- volume level
    tmp = tempfile.mkdtemp(prefix="swec_decode_")
    try:
        base = os.path.join(tmp, "1")
        size, want = lay_down_volume(base, a.gib)
        res["dat_bytes"] = size
        res["shard_bytes"] = os.path.getsize(base + ".ec00")

        def clear():
            for ext in (".dat", ".idx"):
                if os.path.exists(base + ext):
                    os.remove(base + ext)

        def timed(call):
            clear()
            t0 = time.perf_counter()
            out = call()
            return time.perf_counter() - t0, out

        def plain():
            return ec.volume_ec_shards_to_volume(base)

        def checked():
            return ec.ec_shards_to_volume_checked(base)

        timed(plain)                                                   # warm-up of both
        timed(checked)

        def alternate(tag, lost=(), plain_ok=True):
            """plain on every shard (it needs all data shards), checked with `lost` moved away"""
            nonlocal ok
            aside = [(base + ".ec%02d" % i, os.path.join(tmp, "lost%02d" % i)) for i in lost]
            tp, tc = [], []
            rep = None
            for _ in range(a.file_reps):
                dt, _ = timed(plain)
                tp.append(dt)
                if plain_ok:
                    ok = ok and file_digest(base + ".dat") == want
                for p, q in aside:
                    os.rename(p, q)
                dt, rep = timed(checked)
                tc.append(dt)
                ok = ok and file_digest(base + ".dat") == want and rep["ok"] and rep["dat_file_size"] == size
                for p, q in aside:
                    os.rename(q, p)
            res[f"{tag}_plain_s"] = tp
            res[f"{tag}_checked_s"] = tc
            res[f"{tag}_checked_over_plain_best"] = min(tc) / min(tp)
            res[f"{tag}_damaged_columns"] = rep["damaged_columns"]

        alternate("clean")
        alternate("two_lost_3_12", lost=(3, 12))
        shard5 = base + ".ec05"
        with open(shard5, "r+b") as f:                                 # one flipped byte per MiB of data shard 5
            for off in range(12345, os.path.getsize(shard5), 1 << 20):
                f.seek(off)
                b = f.read(1)
                f.seek(off)
                f.write(bytes([b[0] ^ 0x5A]))
        alternate("scattered_damage", plain_ok=False)
        clear()
        plain()
        res["scattered_damage_plain_dat_intact"] = file_digest(base + ".dat") == want
        clear()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)

    # ---- device level
    L = seaweedfs_b200.lib()
    n = int(a.dev_gib * (1 << 30)) & ~4095
    shards = [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(14)]
    for i in range(10):
        seaweedfs_b200._native.check(L.swec_synth_fill_device(0, shards[i].data_ptr(), i * n, n, SEED, None))
    enc = ec.Encoder(10, 4, device=0)
    enc.encode_device([s.data_ptr() for s in shards[:10]], [s.data_ptr() for s in shards[10:]], n)
    enc.synchronize()
    ptrs = [s.data_ptr() for s in shards]
    present = [0] + [1] * 13
    want0 = shards[0].clone()

    def dev_plain():
        enc.reconstruct_device(ptrs, present, n, data_only=True)
        enc.synchronize()

    def dev_checked():
        return enc.decode_data_checked_device(ptrs, present, n)

    for _ in range(2):
        dev_plain()
        ok = ok and dev_checked()["damaged_columns"] == 0
    tp, tc = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        dev_plain()
        tp.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        dev_checked()
        tc.append(time.perf_counter() - t0)
    ok = ok and bool(torch.equal(shards[0], want0))
    res.update({"dev_shard_bytes": n, "dev_plain_s_best": min(tp), "dev_plain_s_median": float(np.median(tp)),
                "dev_checked_s_best": min(tc), "dev_checked_s_median": float(np.median(tc)),
                "dev_checked_over_plain_best": min(tc) / min(tp)})
    res["check"] = "ok" if ok else "MISMATCH"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
