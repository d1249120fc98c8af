"""Speed of the checked sketch locate (swec_locate_sketch_damage_checked, include/swec.h), on one GPU.

The set is a 30 GiB RS(10,4) volume: 14 shards of 786,432 pages.  Synthetic sketch arrays stand for the holders'
sketches: random information words and the parity words rn.encode computes from them (uint8 views) are a clean set,
because sketches are GF(2^8)-linear.  Timed, in one process and after a warm-up of every pattern:
  full      swec_locate_sketch_damage on the full set
  checked0  the checked call on the full set
  checked1  the checked call with one data shard lost (its rebuilt sketch downloaded)
  checked2  the checked call with a data and a parity shard lost (both rebuilt sketches downloaded)
each at radius 1, the calls alternating within every round; best and median of --reps rounds, host clock around the
synchronous call (it uploads the sketches, so the time includes the 14 x 6 MiB host-to-device copies).

Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=786432)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch

    from oracle import rs_numpy as rn
    from seaweedfs_b200 import erasure_coding as ec
    assert torch.cuda.is_available(), "bench_sketch_checked needs a GPU"
    k, m, pages = 10, 4, args.pages
    enc = ec.Encoder(k, m, device=0)
    rng = np.random.default_rng(30)
    data = [rng.integers(0, 256, 8 * pages, dtype=np.uint8) for _ in range(k)]
    true = [d.view("<u8") for d in data] + [p.view("<u8") for p in rn.encode(k, m, data)]
    shard_len = pages * 4096
    patterns = {"checked0": (), "checked1": (3,), "checked2": (3, 12)}

    def full():
        res = enc.locate_sketch_damage(true, shard_len, radius=1)
        assert res["ok"]

    def checked(lost):
        def run():
            res = enc.locate_sketch_damage_checked([None if i in lost else s for i, s in enumerate(true)], shard_len,
                                                   radius=1)
            assert res["ok"] and sorted(res["rebuilt"]) == sorted(lost)
            return res
        return run

    calls = {"full": full, **{name: checked(lost) for name, lost in patterns.items()}}
    for name, lost in patterns.items():   # warm-up, and the predicted sketches are the true ones
        res = calls[name]()
        for i in lost:
            assert (res["rebuilt"][i] == true[i]).all(), (name, i)
    full()
    ts = {name: [] for name in calls}
    for _ in range(args.reps):
        for name, fn in calls.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            ts[name].append(time.perf_counter() - t0)
    out = {"card": card(), "pages": pages, "shards": k + m, "radius": 1}
    for name, v in ts.items():
        out[name] = {"best_ms": 1e3 * min(v), "median_ms": 1e3 * float(np.median(v))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
