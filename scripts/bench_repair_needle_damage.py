"""Cost of repairing a mounted volume in one call (swec_ec_volume_repair_needle_damage) against the three calls it
replaces: swec_ec_volume_locate_needle_damage, swec_repair_ec_damage by path, and swec_ec_volume_scrub_needles to learn
whether the named needles are good again.  A .dat of 10 x --gib GiB of well-formed needle records (4-200 KiB of Data,
CRC32-C computed on the host) is EC-encoded by swec_ec_shards_generate into 14 shard files of --gib GiB, read from the
page cache.  Two sets: clean, and one flipped byte per MiB of data shard 3.  The two arms alternate, --reps times each;
before every call of the damaged set the same bytes are flipped again, so each call starts from the same damaged files
(a repair restores exactly those bytes).  Reports every time, the best of the runs and the median, and the GPU's name,
power limit and maximum SM clock read in the same run.  One JSON line to stdout (and --out).

    python scripts/bench_repair_needle_damage.py [--gib 1] [--reps 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SEED = 0x4E9A12
MIB = 1 << 20
COOKIE = 0x1234ABCD
NEEDLE_KEYS = ("needle_id", "offset", "size", "shard_mask", "damaged_bytes", "uncorrectable_bytes")


def volume_image(dat_size: int, rng):
    """A v3 volume image: superblock, then records of 4-200 KiB of random Data back to back, the tail left random.
    Returns (image, [(id, offset, size)])."""
    import needle_oracle as no
    dat = np.empty(dat_size, dtype=np.uint8)
    for o in range(0, dat_size, 256 * MIB):
        n = min(256 * MIB, dat_size - o)
        dat[o:o + n] = np.frombuffer(rng.bytes(n), dtype=np.uint8)
    dat[:8] = [3, 0, 0, 0, 0, 0, 0, 0]
    lens = rng.integers(4096, 200 * 1024, dat_size // 4096)
    sizes = lens + 5                                           # DataSize, Data, Flags
    actual = (16 + sizes + 4 + 8) // 8 * 8 + 8
    ends = 8 + np.cumsum(actual)
    offs = np.concatenate([[8], ends[:-1]])
    keep = ends <= dat_size
    offs, lens, sizes = offs[keep], lens[keep], sizes[keep]
    recs = []
    for j, (o, n, s) in enumerate(zip(offs.tolist(), lens.tolist(), sizes.tolist())):
        dat[o:o + 16] = np.frombuffer(COOKIE.to_bytes(4, "big") + (j + 1).to_bytes(8, "big") + s.to_bytes(4, "big"), np.uint8)
        dat[o + 16:o + 20] = np.frombuffer(n.to_bytes(4, "big"), np.uint8)
        dat[o + 20 + n] = 0                                    # Flags
        end = o + no.actual_size(s, 3)
        dat[o + 16 + s + 4:end] = 0                            # timestamp 0, padding
        recs.append((j + 1, o, s))
    crcs = no.ranges_crc32c(dat, offs + 20, lens)
    for (_, o, s), c in zip(recs, crcs.tolist()):
        dat[o + 16 + s:o + 20 + s] = np.frombuffer(int(c).to_bytes(4, "big"), np.uint8)
    return dat, recs


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()

    from oracle import rs_numpy as rn
    from seaweedfs_b200 import erasure_coding as ec

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    n = int(a.gib * (1 << 30)) // MIB * MIB
    dat_size = 10 * n                          # below 10 GiB: small rows only
    res = {"gpu": gpu, "shard_bytes": n}
    tmp = tempfile.mkdtemp(prefix="swec_repair_needle_damage_")
    try:
        if shutil.disk_usage(tmp).free < dat_size + 14 * n + (1 << 30):
            res["check"] = "not measured: too little free disk"
            print(json.dumps(res))
            return
        base = os.path.join(tmp, "1")
        t0 = time.perf_counter()
        dat, recs = volume_image(dat_size, np.random.default_rng(SEED))
        dat.tofile(base + ".dat")
        del dat
        open(base + ".idx", "wb").write(b"".join(rn._entry(i, o // 8, s) for i, o, s in recs))
        ec.volume_ec_shards_generate(base, needle_version=3)
        os.remove(base + ".dat")
        res.update({"records": len(recs), "setup_s": time.perf_counter() - t0})
        flips = list(range(12345, n, MIB))     # one byte per MiB of data shard 3

        def damage():
            with open(base + ".ec03", "r+b") as f:
                for o in flips:
                    f.seek(o)
                    b = f.read(1)[0]
                    f.seek(o)
                    f.write(bytes([b ^ 0x40]))

        vol = ec.EcVolume(base)
        ok = True

        def one_call(damaged):
            if damaged:
                damage()
            t = time.perf_counter()
            got = vol.repair_needle_damage(max_needles=1 << 20)
            return time.perf_counter() - t, got

        def three_calls(damaged):
            if damaged:
                damage()
            t = time.perf_counter()
            loc = vol.locate_needle_damage(max_needles=1 << 20)
            rep = ec.repair_ec_damage(base)
            _, _, errors = vol.scrub_needles(1)
            return time.perf_counter() - t, (loc, rep, errors)

        def alternate(tag, damaged):
            nonlocal ok
            one, three = [], []
            for _ in range(a.reps):
                t1, got = one_call(damaged)
                t3, (loc, rep, errors) = three_calls(damaged)
                one.append(t1)
                three.append(t3)
                bad = [e for e in errors if re.match(r"needle \d+ on volume", e)]
                named = [{k: v for k, v in r.items() if k in NEEDLE_KEYS} for r in got["needles"]]
                ok = ok and got["ok"] and rep["ok"] and not bad and named == loc["needles"]
                ok = ok and all(r["status"] == 0 for r in got["needles"])
            res.update({f"{tag}_one_call_s": one, f"{tag}_three_calls_s": three,
                        f"{tag}_one_call_best_s": min(one), f"{tag}_three_calls_best_s": min(three),
                        f"{tag}_one_call_median_s": float(np.median(one)),
                        f"{tag}_three_calls_median_s": float(np.median(three)),
                        f"{tag}_speedup_best": min(three) / min(one),
                        f"{tag}_speedup_median": float(np.median(three) / np.median(one))})
            return got

        got = alternate("clean", False)
        ok = ok and got["n_needles"] == 0 and got["damaged_columns"] == 0
        got = alternate("one_byte_per_MiB", True)
        ok = ok and got["shards"] == {3: (len(flips), flips[0], flips[-1])}
        ok = ok and sum(r["damaged_bytes"] for r in got["needles"]) + got["unowned"][0] == len(flips)
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
