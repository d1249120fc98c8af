"""Speed of naming the needles that sketch-located pages hit, and of the holder's sketch through the mounted volume.

  attribute  swec_sketch_needle_damage at full size: the 30 GiB geometry (RS(10,4), 1 GiB / 1 MiB blocks, 3 GiB
             shards) with ~1 M live records; 64 flagged pages, then every page of one data shard flagged (786,432
             pages).  Best and median of 5 host-timed calls (each ends in a device synchronise; the records' upload
             and the counters' read-back are part of the call).
  sketch     swec_ec_volume_page_sketch of 4 local 1 GiB shards (one pipeline pass) against 4 swec_page_sketch_file
             calls on the same files, alternating the arms, best and median of 5 each, files in the page cache.

Prints one JSON line with the card's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_page_sketch import card  # noqa: E402


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts), float(np.median(ts))


def records(rng, dat_size):
    """(needle_id, offset, size) of ~1 M back-to-back version-3 records of 0..60,000 bytes after the superblock."""
    sizes = rng.integers(0, 60_000, 1_100_000)
    actual = 16 + sizes + 4 + 8
    actual += 8 - actual % 8
    offs = 8 + np.concatenate([[0], np.cumsum(actual)[:-1]])
    keep = offs + actual <= dat_size
    return list(zip(range(1, int(keep.sum()) + 1), offs[keep].tolist(), sizes[keep].tolist()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--shard-gib", type=float, default=1.0)
    args = ap.parse_args()
    import ctypes as C

    import torch

    from seaweedfs_b200 import erasure_coding as ec
    from seaweedfs_b200 import lib
    from seaweedfs_b200._native import NeedleDamage, check
    assert torch.cuda.is_available(), "bench_sketch_needle_damage needs a GPU"
    out = {"card": card()}
    L = lib()

    # ---- attribute: the C call with prepared ctypes arrays, so that the Python list handling is not timed
    k, m, large, small, dat_size = 10, 4, 1 << 30, 1 << 20, 30 << 30
    shard_len = ec.expected_shard_size(dat_size, k, large, small)
    n_pages = (shard_len + 4095) // 4096
    rng = np.random.default_rng(7)
    recs = records(rng, dat_size)
    arr = (NeedleDamage * len(recs))()
    for r, (nid, off, size) in zip(arr, recs):
        r.needle_id, r.offset, r.size = nid, off, size
    unowned = (C.c_uint64 * 2)()
    runs = {}
    for name, pages in (("64_pages", sorted((int(g), 1 << 3, False) for g in rng.choice(n_pages, 64, replace=False))),
                        ("one_shard_every_page", [(g, 1 << 3, False) for g in range(n_pages)])):
        parr, n = ec._sketch_pages(pages)

        def call():
            check(L.swec_sketch_needle_damage(0, k, m, shard_len, dat_size, large, small, parr, n, arr, len(recs),
                                              unowned))
        call()
        best, med = timed(call, args.reps)
        runs[name] = {"pages": n, "best_s": best, "median_s": med,
                      "damaged_bytes": sum(int(r.damaged_bytes) for r in arr) + int(unowned[0])}
    out["attribute"] = {"records": len(recs), "shard_len": shard_len, **runs}

    # ---- sketch: 4 local shards through the handle against 4 file calls
    size = int(args.shard_gib * (1 << 30))
    with tempfile.TemporaryDirectory() as d:
        base = os.path.join(d, "1")
        data = np.random.default_rng(1).integers(0, 256, size, dtype=np.uint8)
        for i in range(4):
            np.roll(data, i * 4096).tofile(base + ".ec%02d" % i)
        open(base + ".ecx", "wb").close()
        vol = ec.EcVolume(base)
        ids = list(range(4))
        want = {i: ec.page_sketch_file(base + ".ec%02d" % i, 99)[0] for i in ids}   # also warms the page cache
        got, _ = vol.page_sketch(99, ids)
        assert all(np.array_equal(got[i], want[i]) for i in ids)
        t_handle, t_files = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            vol.page_sketch(99, ids)
            t_handle.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            for i in ids:
                ec.page_sketch_file(base + ".ec%02d" % i, 99)
            t_files.append(time.perf_counter() - t0)
        vol.close()
    total = 4 * size
    out["sketch"] = {"shards": 4, "shard_bytes": size,
                     "handle_best_s": min(t_handle), "handle_median_s": float(np.median(t_handle)),
                     "files_best_s": min(t_files), "files_median_s": float(np.median(t_files)),
                     "handle_best_gbps": total / min(t_handle) / 1e9, "files_best_gbps": total / min(t_files) / 1e9}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
