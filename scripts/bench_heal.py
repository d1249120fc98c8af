"""Speed of the heal (swec_heal_ec_files, swec_heal_device; include/swec.h) against the two-call flow it replaces, on one
GPU: the checked rebuild, then the repair of the completed set.

  file arm    14 shard files of --file-gib GiB (RS(10,4)) in the page cache, parity shard 12 lost, one flipped byte
              per MiB of data shard 3: heal_ec_files against rebuild_ec_files_checked + repair_ec_damage
  device arm  14 shards of --dev-gib GiB in HBM, the same loss and damage: heal_device against
              reconstruct_checked_device + correct_damage_device

Before every call the damage is applied again (the calls correct it) and the rebuilt shard is removed; every call's
report is checked.  The two flows alternate within each round, after a warm-up round of both; best and median of
--reps rounds, host clock around the synchronous calls.  Prints one JSON line with the card's name, power limit and
SM clock, read in the same run.
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

K, M, LOST, DAMAGED = 10, 4, 12, 3
MIB = 1 << 20


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def stats(v):
    return {"best_s": min(v), "median_s": float(np.median(v))}


def rounds(arms, reps):
    for fn in arms.values():      # warm-up: run-time kernels compiled, staging rings pinned
        fn()
    ts = {name: [] for name in arms}
    for _ in range(reps):
        for name, fn in arms.items():
            ts[name].append(fn())
    return {name: stats(v) for name, v in ts.items()}


def file_arm(torch, ec, gib, reps, where):
    n = gib << 30
    d = tempfile.mkdtemp(prefix="bench_heal_", dir=where)
    try:
        base = os.path.join(d, "1")
        shards = [torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda") for _ in range(K)]
        shards += [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(M)]
        enc = ec.Encoder(K, M, device=0)
        enc.encode_device([s.data_ptr() for s in shards[:K]], [s.data_ptr() for s in shards[K:]], n)
        enc.synchronize()
        for i, s in enumerate(shards):
            if i != LOST:
                s.cpu().numpy().tofile(base + ".ec%02d" % i)
        del shards
        torch.cuda.empty_cache()
        offs = np.arange(0, n, MIB) + 4097

        def damage():
            with open(base + ".ec%02d" % DAMAGED, "r+b") as f:
                for o in offs:
                    f.seek(int(o))
                    b = f.read(1)
                    f.seek(int(o))
                    f.write(bytes([b[0] ^ 0x5A]))
            if os.path.exists(base + ".ec%02d" % LOST):
                os.remove(base + ".ec%02d" % LOST)

        def heal():
            damage()
            t0 = time.perf_counter()
            rep = ec.heal_ec_files(base)
            t = time.perf_counter() - t0
            assert rep["ok"] and rep["rebuilt"] == [LOST] and rep["shards"] == {DAMAGED: (len(offs), 4097, int(offs[-1]))}
            return t

        def two_calls():
            damage()
            t0 = time.perf_counter()
            rep = ec.rebuild_ec_files_checked(base)
            rep2 = ec.repair_ec_damage(base)
            t = time.perf_counter() - t0
            assert rep["ok"] and rep["rebuilt"] == [LOST] and rep["damaged_columns"] == len(offs)
            assert rep2["ok"] and rep2["shards"] == {DAMAGED: (len(offs), 4097, int(offs[-1]))}
            return t

        out = rounds({"heal": heal, "checked_then_repair": two_calls}, reps)
        out.update({"shard_gib": gib, "dir": where, "flipped_bytes": len(offs)})
        return out
    finally:
        shutil.rmtree(d, ignore_errors=True)


def device_arm(torch, ec, gib, reps):
    n = gib << 30
    shards = [torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda") for _ in range(K)]
    shards += [torch.empty(n, dtype=torch.uint8, device="cuda") for _ in range(M)]
    enc = ec.Encoder(K, M, device=0)
    ptrs = [s.data_ptr() for s in shards]
    enc.encode_device(ptrs[:K], ptrs[K:], n)
    enc.synchronize()
    present = [i != LOST for i in range(K + M)]
    idx = torch.arange(4097, n, MIB, device="cuda")
    want = {DAMAGED: (idx.numel(), 4097, int(idx[-1]))}

    def damage():
        shards[DAMAGED][idx] ^= 0x5A
        shards[LOST].zero_()
        torch.cuda.synchronize()

    def heal():
        damage()
        t0 = time.perf_counter()
        rep = enc.heal_device(ptrs, present, n)
        t = time.perf_counter() - t0
        assert rep["shards"] == want and rep["uncorrectable_columns"] == 0
        return t

    def two_calls():
        damage()
        t0 = time.perf_counter()
        rep = enc.reconstruct_checked_device(ptrs, present, n)
        rep2 = enc.correct_damage_device(ptrs, n)
        t = time.perf_counter() - t0
        assert rep["shards"] == want and rep2["shards"] == want
        return t

    out = rounds({"heal": heal, "checked_then_correct": two_calls}, reps)
    out["shard_gib"] = gib
    del shards
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--file-gib", type=int, default=1)
    ap.add_argument("--dev-gib", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dir", default=None, help="where the shard files go (default: the temporary directory)")
    args = ap.parse_args()
    import torch

    from seaweedfs_b200 import erasure_coding as ec
    assert torch.cuda.is_available(), "bench_heal needs a GPU"
    out = {"card_before": card(), "reps": args.reps}
    out["device"] = device_arm(torch, ec, args.dev_gib, args.reps)
    out["file"] = file_arm(torch, ec, args.file_gib, args.reps, args.dir or tempfile.gettempdir())
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
