"""Rate of the GPU needle check (swec_check_needles_device) over a 30 GiB volume image in HBM, against the host's
CRC32-C (SSE4.2) on one core and on all cores over the same records.

The image is the seeded synthetic stream with needle headers and tails written over it (the record mix of the
full-size test: sizes log-uniform from 1 B to 8 MiB, empty and 1-64 B records, a 1.5 GiB record).  Bytes read are
the whole image: every record's header, body and tail.  One JSON line to stdout (and --out).

    python scripts/bench_needle_check.py [--gib 30] [--reps 10] [--host-gib 4] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_PEAK = 3.35e12  # H100 SXM data sheet


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=30)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--host-gib", type=float, default=4)
    ap.add_argument("--out")
    a = ap.parse_args()

    import torch

    import needle_oracle as no
    import seaweedfs_b200
    from seaweedfs_b200 import erasure_coding as ec
    from test_needles import SEED, lay_records, synthetic_image

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    size = int(a.gib * (1 << 30)) & ~7
    rng = np.random.default_rng(1003)
    recs, extras = synthetic_image(3, size, 1536 << 20, rng)
    crcs = no.synth_crc32c(SEED, [r[3] for r in recs], [r[4] for r in recs])
    img = torch.empty(size, dtype=torch.uint8, device="cuda")
    seaweedfs_b200._native.check(seaweedfs_b200.lib().swec_synth_fill_device(0, img.data_ptr(), 0, size, SEED, None))
    img[0] = 3
    lay_records(torch, img, 3, recs, extras, crcs)
    torch.cuda.synchronize()
    entries = [(k, off, s) for k, off, s, _, _ in recs]
    image_bytes = recs[-1][1] + no.actual_size(recs[-1][2], 3) - recs[0][1]
    data_bytes = sum(r[4] for r in recs)

    out = ec.check_needles_device(img.data_ptr(), size, entries, needle_version=3, device=0)  # warm-up + check
    ok = all(r["status"] == 0 and r["crc_want"] == int(c) for r, c in zip(out, crcs))
    from seaweedfs_b200._native import NeedleCheck
    arr = (NeedleCheck * len(entries))()
    for c, (k, off, s) in zip(arr, entries):
        c.needle_id, c.offset, c.size = k, off, s
    L = seaweedfs_b200.lib()
    times = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        seaweedfs_b200._native.check(L.swec_check_needles_device(0, img.data_ptr(), size, 3, arr, len(entries), None))
        times.append(time.perf_counter() - t0)   # the call synchronises its stream
    best, med = min(times), float(np.median(times))

    # the host over the same kind of records: the first --host-gib of the image, copied to host memory
    hsize = min(size, int(a.host_gib * (1 << 30)))
    host = img[:hsize].cpu().numpy()
    del img
    torch.cuda.empty_cache()
    hr = [r for r in recs if r[3] + r[4] <= hsize]
    hoff, hlen = [r[3] for r in hr], [r[4] for r in hr]
    hbytes = sum(hlen)
    rates = {}
    for threads in (1, os.cpu_count() or 1):
        no.ranges_crc32c(host, hoff[:50], hlen[:50], threads=threads)
        t0 = time.perf_counter()
        got = no.ranges_crc32c(host, hoff, hlen, threads=threads)
        rates[threads] = hbytes / (time.perf_counter() - t0)
        ok = ok and all(int(g) == int(c) for g, c in zip(got, crcs[:len(hr)]))

    res = {"gpu": gpu, "records": len(recs), "image_bytes": image_bytes, "data_bytes": data_bytes,
           "check_s_best": best, "check_s_median": med,
           "gpu_GBps_best": image_bytes / best / 1e9, "gpu_GBps_median": image_bytes / med / 1e9,
           "fraction_of_3.35TBps_best": image_bytes / best / HBM_PEAK,
           "host_cores": os.cpu_count(), "host_sse42": bool(no.host().orc_crc32c_has_hw()),
           "host_1core_GBps": rates[1] / 1e9, "host_all_cores_GBps": rates[max(rates)] / 1e9,
           "host_bytes": hbytes, "check": "ok" if ok else "MISMATCH"}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
