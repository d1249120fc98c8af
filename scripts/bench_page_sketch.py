"""Speed of the page sketch calls (include/swec.h, SWEC_PAGE_SKETCH_VERSION), on one GPU.

  device   swec_page_sketch_device over a 3 GiB shard in HBM, best and median of 10, beside swec_digest_device (a
           plain streaming read of the same buffer) in the same process
  file     swec_page_sketch_file over a 1 GiB shard file in the page cache (read once before timing), best of 3
  locate   swec_locate_sketch_damage over 14 x 786,432 pages (an RS(10,4) set of 3 GiB shards): a clean set, and one
           with 64 damaged pages

Prints one JSON line with the card's name and power limit.  The bar: the device rate is at least 4x the file rate, so
that the file call is bound by its reads rather than by the kernel.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
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
    ap.add_argument("--device-gib", type=float, default=3.0)
    ap.add_argument("--file-gib", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    import torch

    from seaweedfs_b200 import erasure_coding as ec
    from seaweedfs_b200 import lib
    assert torch.cuda.is_available(), "bench_page_sketch needs a GPU"
    L = lib()
    enc = ec.Encoder(10, 4, device=0)
    out = {"card": card()}

    # ---- device
    n = int(args.device_gib * (1 << 30))
    buf = torch.empty(n, dtype=torch.uint8, device="cuda")
    assert L.swec_synth_fill_device(0, buf.data_ptr(), 0, n, 0x5EED, None) == 0
    pages = (n + 4095) // 4096
    sk = torch.empty(pages, dtype=torch.int64, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(args.reps):
            ev[0].record()
            fn()
            ev[1].record()
            torch.cuda.synchronize()
            ts.append(ev[0].elapsed_time(ev[1]) / 1e3)
        return min(ts), float(np.median(ts))

    stream = torch.cuda.current_stream().cuda_stream
    best, med = timed(lambda: enc.page_sketch_device(buf.data_ptr(), n, sk.data_ptr(), 0x1234, 0, stream))
    out["device_sketch"] = {"bytes": n, "best_s": best, "median_s": med, "best_gbps": n / best / 1e9,
                            "median_gbps": n / med / 1e9}
    import ctypes as C
    dg = C.c_uint64(0)
    best, med = timed(lambda: L.swec_digest_device(0, buf.data_ptr(), n, C.byref(dg), stream))
    out["digest"] = {"bytes": n, "best_s": best, "median_s": med, "best_gbps": n / best / 1e9,
                     "median_gbps": n / med / 1e9}

    # ---- file
    fn = int(args.file_gib * (1 << 30))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "1.ec00")
        host = buf[:fn].cpu().numpy()
        host.tofile(path)
        with open(path, "rb") as f:
            while f.read(64 << 20):
                pass
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            got, length = ec.page_sketch_file(path, 0x1234)
            ts.append(time.perf_counter() - t0)
        assert length == fn and (got == sk[:len(got)].cpu().numpy().view(np.uint64)).all()
    out["file_sketch"] = {"bytes": fn, "best_s": min(ts), "best_gbps": fn / min(ts) / 1e9}
    out["device_over_file"] = out["device_sketch"]["best_gbps"] / out["file_sketch"]["best_gbps"]

    # ---- locate over the sketches of an RS(10,4) set of 3 GiB shards
    npages = 786432
    rng = np.random.default_rng(1)
    sketches = [rng.integers(0, 1 << 63, npages, dtype=np.uint64) for _ in range(10)]
    sketches += [np.zeros(npages, dtype=np.uint64) for _ in range(4)]
    enc.encode([s.view(np.uint8) for s in sketches])
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        res = enc.locate_sketch_damage(sketches, npages * 4096)
        ts.append(time.perf_counter() - t0)
    assert res["ok"]
    bad = [s.copy() for s in sketches]
    for g in rng.choice(npages, 64, replace=False):
        bad[int(g) % 14][g] ^= np.uint64(0xA5)
    t0 = time.perf_counter()
    res = enc.locate_sketch_damage(bad, npages * 4096)
    t_bad = time.perf_counter() - t0
    assert res["n_flagged"] == 64 and not any(u for _, _, u in res["pages"])
    out["locate"] = {"pages": npages, "shards": 14, "clean_best_s": min(ts), "damaged_64_s": t_bad}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
