"""The argument rules of the fourteen damage entry points, as exact (status, swec_last_error()) pairs.

Every call here fails before any device work: the encoders and the mounted volume are opened with device < 0, so the
first combination that passes every rule reaches SWEC_ERR_NO_DEVICE.  Each rule is checked alone, pairs of violations
pin which rule wins, and the texts are part of what is checked: a caller may show them, and the Go and Python bindings
pass them on unchanged.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_needle_damage as tnd  # noqa: E402

from seaweedfs_b200._native import DamageRange, DamageReport, NeedleCheck, NeedleDamage, SketchPage  # noqa: E402

BAD, FEW, NODEV = -1, -2, -7
NULL_ARG = "NULL argument"
NO_REPORT = "report is NULL"
CAP = "ranges_cap must be >= 0, and ranges non-NULL when it is > 0"
R12 = "radius must be 1 or 2"
R012 = "radius must be 0, 1 or 2"
PAGES_CAP = "pages_cap must be >= 0, and pages non-NULL when it is > 0"
NEEDLES = "needles_cap must be >= 0, and needles non-NULL when it is > 0"
UNOWNED = "unowned is NULL"
RECORDS = "n_records must be >= 0, and records non-NULL when it is > 0"
CHECKS = "checks must be non-NULL when needles_cap is > 0"
ENC_NODEV = "encoder was created without a device (device < 0); no CPU fallback exists"
VOL_NODEV = "no CUDA device: the volume was opened with device < 0"


def parity(r, m):
    return f"radius {r} needs at least {2 * r} parity shards, the code has {m}"


class Env:
    """Device-less encoders of RS(10,4) and RS(3,2), a CPU-made RS(10,4) volume and one of RS(3,2), and the buffers
    the calls point at (never read: every call fails before it would)."""

    def __init__(self, swec, root):
        self.L = swec.lib()
        ec = swec.erasure_coding
        self.enc = {4: ec.Encoder(10, 4, device=-1), 2: ec.Encoder(3, 2, device=-1)}
        self.base = {4: tnd.cpu_volume(root, name="v4"), 2: tnd.cpu_volume(root, k=3, m=2, name="v2")}
        self.dat_size = {m: int(json.load(open(b + ".vif"))["datFileSize"]) for m, b in self.base.items()}
        self.root = str(root)
        self.words = [np.zeros(4096, dtype=np.uint64) for _ in range(14)]
        self.report, self.ranges, self.n = DamageReport(), (DamageRange * 4)(), C.c_int(0)
        self.ok, self.n_rebuilt, self.ids = C.c_int(0), C.c_int(0), (C.c_uint32 * 32)()
        self.needles, self.checks, self.n_needles = (NeedleDamage * 4)(), (NeedleCheck * 4)(), C.c_int(0)
        self.unowned, self.size = (C.c_uint64 * 2)(), C.c_int64(0)
        self.pages, self.n_flagged, self.per_shard = (SketchPage * 4)(), C.c_int64(0), (C.c_uint64 * 32)()
        self.vols = []

    def out(self, report=True, ranges=True, cap=4, n_ranges=True):
        """The report out-parameters: report, ranges, ranges_cap, n_ranges."""
        return (C.byref(self.report) if report else None, self.ranges if ranges else None, cap,
                C.byref(self.n) if n_ranges else None)

    def ptrs(self, n, null=()):
        return (C.c_void_p * n)(*[None if i in null else self.words[i].ctypes.data for i in range(n)])

    def present(self, n, lost=()):
        return np.array([0 if i in lost else 1 for i in range(n)], dtype=np.uint8)

    def volume(self, m):
        from seaweedfs_b200.erasure_coding import EcVolume
        v = EcVolume(self.base[m], device=-1)
        self.vols.append(v)
        return v

    def close(self):
        for v in self.vols:
            v.close()


def p(v, on):
    return C.byref(v) if on else None


# ---- one caller per entry point: every argument valid unless overridden -------------------------------------------

def device_call(name):
    def call(env, m=4, e=True, shards=True, null=(), radius=1, **out):
        enc = env.enc[m]
        t = enc.total_shards
        return getattr(env.L, name)(enc._h if e else None, env.ptrs(t, null) if shards else None, 4096, radius,
                                    *env.out(**out), None)
    return call


def checked_device_call(name):
    def call(env, m=4, e=True, shards=True, null=(), present=True, lost=(), radius=1, **out):
        enc = env.enc[m]
        t = enc.total_shards
        pres = env.present(t, lost)
        return getattr(env.L, name)(enc._h if e else None, env.ptrs(t, null) if shards else None,
                                    pres.ctypes.data if present else None, 4096, radius, *env.out(**out), None)
    return call


def files_call(name):
    def call(env, m=4, base=True, dirs=False, ok=True, km=True, radius=1, **out):
        k = 10 if m == 4 else 3
        b = env.base[m if m in env.base else 4].encode() if base else None
        return getattr(env.L, name)(b, None, 1 if dirs else 0, k if km else 0, m if km else 0, -1, radius,
                                    *env.out(**out), p(env.ok, ok))
    return call


def rebuild_checked(env, m=4, base=True, rebuilt=True, n_rebuilt=True, ok=True, radius=1, **out):
    k = 10 if m == 4 else 3
    return env.L.swec_rebuild_ec_files_checked(env.base[m].encode() if base else None, None, 0, k, m, -1, radius,
                                               env.ids if rebuilt else None, p(env.n_rebuilt, n_rebuilt),
                                               *env.out(**out), p(env.ok, ok))


def write_dat_checked(env, m=4, base=True, names=True, ok=True, lost=(), k=None, radius=1, **out):
    kk = 10 if m == 4 else 3
    arr = (C.c_char_p * (kk + m))(*[None if i in lost else (env.base[m] + ".ec%02d" % i).encode()
                                    for i in range(kk + m)])
    return env.L.swec_write_dat_file_checked((env.root + "/out").encode() if base else None, env.dat_size[m],
                                             arr if names else None, kk if k is None else k, m, 1 << 30, 1 << 20, -1,
                                             radius, *env.out(**out), p(env.ok, ok))


def to_volume_checked(env, m=4, base=True, ok=True, radius=1, **out):
    return env.L.swec_ec_shards_to_volume_checked(env.base[m].encode() if base else None, None, None, 0, -1, radius,
                                                  C.byref(env.size), *env.out(**out), p(env.ok, ok))


def needle_device(env, m=4, e=True, shards=True, null=(), radius=1, records=True, n_records=1, unowned=True,
                  dat_size=4096, **out):
    enc = env.enc[m]
    return env.L.swec_locate_needle_damage_device(enc._h if e else None, env.ptrs(enc.total_shards, null) if shards else None,
                                                  4096, dat_size, 1 << 30, 1 << 20, radius,
                                                  env.needles if records else None, n_records, *env.out(**out),
                                                  env.unowned if unowned else None, None)


def handle_locate(env, m=4, v=True, radius=1, needles=True, needles_cap=4, n_needles=True, unowned=True, ok=True,
                  **out):
    h = env.volume(m)._h if v else None
    return env.L.swec_ec_volume_locate_needle_damage(h, radius, *env.out(**out), env.needles if needles else None,
                                                     needles_cap, p(env.n_needles, n_needles),
                                                     env.unowned if unowned else None, p(env.ok, ok))


def handle_repair(env, m=4, v=True, radius=1, needles=True, checks=True, needles_cap=4, n_needles=True, unowned=True,
                  ok=True, **out):
    h = env.volume(m)._h if v else None
    return env.L.swec_ec_volume_repair_needle_damage(h, radius, *env.out(**out), env.needles if needles else None,
                                                     env.checks if checks else None, needles_cap,
                                                     p(env.n_needles, n_needles), env.unowned if unowned else None,
                                                     p(env.ok, ok))


def sketch_call(checked):
    def call(env, m=4, e=True, sketches=True, lost=(), shard_len=8192, radius=1, pages=True, pages_cap=4,
             n_flagged=True, ok=True):
        enc = env.enc[m]
        sk = env.ptrs(enc.total_shards, lost) if sketches else None
        args = [enc._h if e else None, sk, shard_len, radius, env.pages if pages else None, pages_cap,
                p(env.n_flagged, n_flagged), env.per_shard]
        if checked:
            args.append(None)
        return getattr(env.L, "swec_locate_sketch_damage_checked" if checked else "swec_locate_sketch_damage")(
            *args, p(env.ok, ok))
    return call


CALLS = {
    "locate_damage_device": device_call("swec_locate_damage_device"),
    "correct_damage_device": device_call("swec_correct_damage_device"),
    "reconstruct_checked_device": checked_device_call("swec_reconstruct_checked_device"),
    "decode_data_checked_device": checked_device_call("swec_decode_data_checked_device"),
    "locate_ec_damage": files_call("swec_locate_ec_damage"),
    "repair_ec_damage": files_call("swec_repair_ec_damage"),
    "rebuild_ec_files_checked": rebuild_checked,
    "write_dat_file_checked": write_dat_checked,
    "ec_shards_to_volume_checked": to_volume_checked,
    "locate_needle_damage_device": needle_device,
    "ec_volume_locate_needle_damage": handle_locate,
    "ec_volume_repair_needle_damage": handle_repair,
    "locate_sketch_damage": sketch_call(False),
    "locate_sketch_damage_checked": sketch_call(True),
}

# The report rules, alone and against each other, shared by every call that takes a report.
REPORT_RULES = [
    ("no-report", dict(report=False), BAD, NO_REPORT),
    ("negative-cap", dict(cap=-1), BAD, CAP),
    ("no-ranges", dict(ranges=False), BAD, CAP),
    ("no-ranges-cap-0", dict(ranges=False, cap=0), None, None),      # valid: reaches what follows
    ("no-n-ranges", dict(n_ranges=False), None, None),               # valid: n_ranges may be NULL
    ("no-report-negative-cap", dict(report=False, cap=-1), BAD, NO_REPORT),
]
# radius 1 or 2 and 2·radius <= m, checked after the report
LOCATE_RADIUS = [
    ("radius-0", dict(radius=0), BAD, R12),
    ("radius-3", dict(radius=3), BAD, R12),
    ("radius-minus-1", dict(radius=-1), BAD, R12),
    ("radius-2-m-2", dict(radius=2, m=2), BAD, parity(2, 2)),
    ("radius-2-m-4", dict(radius=2), None, None),
    ("radius-1-m-2", dict(radius=1, m=2), None, None),
    ("no-report-radius-3", dict(report=False, radius=3), BAD, NO_REPORT),
    ("negative-cap-radius-3", dict(cap=-1, radius=3), BAD, CAP),
    ("no-report-radius-2-m-2", dict(report=False, radius=2, m=2), BAD, NO_REPORT),
    ("no-ranges-radius-2-m-2", dict(ranges=False, radius=2, m=2), BAD, CAP),
]
# radius 0, 1 or 2, with no parity rule (the checked calls clamp it to what the present shards allow)
REBUILD_RADIUS = [
    ("radius-0", dict(radius=0), None, None),
    ("radius-2-m-2", dict(radius=2, m=2), None, None),
    ("radius-3", dict(radius=3), BAD, R012),
    ("radius-minus-1", dict(radius=-1), BAD, R012),
    ("no-report-radius-3", dict(report=False, radius=3), BAD, NO_REPORT),
    ("negative-cap-radius-3", dict(cap=-1, radius=3), BAD, CAP),
]


def cases():
    """(id, call, overrides, status, text); a None status is filled in with the call's first valid outcome."""
    out = []

    def add(call, rows, valid):
        for name, over, st, text in rows:
            out.append((f"{call}-{name}", call, over, *((st, text) if st is not None else valid)))

    # the device calls: the encoder and shard pointers first, then the report, the radius, each shard, the device
    for call in ("locate_damage_device", "correct_damage_device"):
        valid = (NODEV, ENC_NODEV)
        add(call, REPORT_RULES + LOCATE_RADIUS + [
            ("no-encoder", dict(e=False), BAD, NULL_ARG),
            ("no-shards", dict(shards=False), BAD, NULL_ARG),
            ("no-encoder-no-report", dict(e=False, report=False), BAD, NULL_ARG),
            ("null-shard", dict(null=(13,)), BAD, "NULL shard"),
            ("null-shard-radius-3", dict(null=(13,), radius=3), BAD, R12),
            ("null-shard-no-report", dict(null=(0,), report=False), BAD, NO_REPORT),
            ("valid", {}, *valid),
        ], valid)
    for call in ("reconstruct_checked_device", "decode_data_checked_device"):
        valid = (NODEV, ENC_NODEV)
        decode = call.startswith("decode")
        add(call, REPORT_RULES + REBUILD_RADIUS + [
            ("no-encoder", dict(e=False), BAD, NULL_ARG),
            ("no-present", dict(present=False), BAD, NULL_ARG),
            ("no-present-no-report", dict(present=False, report=False), BAD, NULL_ARG),
            ("too-few", dict(lost=(0, 1, 2, 3, 4)), FEW, "fewer than data_shards shards present"),
            ("too-few-radius-3", dict(lost=(0, 1, 2, 3, 4), radius=3), BAD, R012),
            ("too-few-null-shard", dict(lost=(0, 1, 2, 3, 4), null=(5,)), FEW, "fewer than data_shards shards present"),
            ("null-present-shard", dict(null=(2,)), BAD, "NULL shard"),
            ("null-lost-data-shard", dict(lost=(2,), null=(2,)), BAD, "missing shard has no buffer"),
            ("null-lost-parity-shard", dict(lost=(12,), null=(12,)),
             *(valid if decode else (BAD, "missing shard has no buffer"))),
            ("null-present-parity-shard", dict(null=(12,)), BAD, "NULL shard"),
            ("four-lost", dict(lost=(0, 5, 11, 13)), *valid),
            ("valid", {}, *valid),
        ], valid)
    # the shard files: base and ok first, then the report and radius against the code's m, then the files
    for call in ("locate_ec_damage", "repair_ec_damage"):
        valid = (NODEV, ENC_NODEV)
        add(call, REPORT_RULES + LOCATE_RADIUS + [
            ("no-base", dict(base=False), BAD, NULL_ARG),
            ("no-ok", dict(ok=False), BAD, NULL_ARG),
            ("dirs-null", dict(dirs=True), BAD, NULL_ARG),
            ("no-ok-no-report", dict(ok=False, report=False), BAD, NULL_ARG),
            ("ratio-from-vif", dict(km=False), *valid),
            ("ratio-from-vif-radius-2-m-2", dict(km=False, m=2, radius=2), BAD, parity(2, 2)),
            ("m-0", dict(m=0), BAD, parity(1, 0)),
            ("m-minus-1", dict(m=-1), BAD, parity(1, -1)),
            ("m-0-radius-2", dict(m=0, radius=2), BAD, parity(2, 0)),
            ("valid", {}, *valid),
        ], valid)
    add("rebuild_ec_files_checked", REPORT_RULES + REBUILD_RADIUS + [
        ("no-base", dict(base=False), BAD, NULL_ARG),
        ("no-rebuilt", dict(rebuilt=False), BAD, NULL_ARG),
        ("no-n-rebuilt", dict(n_rebuilt=False), BAD, NULL_ARG),
        ("no-ok", dict(ok=False), BAD, NULL_ARG),
        ("no-ok-radius-3", dict(ok=False, radius=3), BAD, NULL_ARG),
        ("valid", {}, NODEV, ENC_NODEV),
    ], (NODEV, ENC_NODEV))
    add("write_dat_file_checked", REPORT_RULES + REBUILD_RADIUS + [
        ("no-base", dict(base=False), BAD, "bad argument"),
        ("no-names", dict(names=False), BAD, "bad argument"),
        ("no-ok", dict(ok=False), BAD, "bad argument"),
        ("k-0", dict(k=0), BAD, "bad argument"),
        ("no-ok-no-report", dict(ok=False, report=False), BAD, "bad argument"),
        ("too-few", dict(lost=(0, 1, 2, 3, 4)), FEW,
         "not enough shards to decode {root}/out: found 9 shards, need at least 10"),
        ("too-few-radius-3", dict(lost=(0, 1, 2, 3, 4), radius=3), BAD, R012),
        ("valid", {}, NODEV, ENC_NODEV),
    ], (NODEV, ENC_NODEV))
    add("ec_shards_to_volume_checked", REPORT_RULES + REBUILD_RADIUS + [
        ("no-base", dict(base=False), BAD, NULL_ARG),
        ("no-ok", dict(ok=False), BAD, NULL_ARG),
        ("no-ok-radius-3", dict(ok=False, radius=3), BAD, NULL_ARG),
        ("valid", {}, NODEV, ENC_NODEV),
    ], (NODEV, ENC_NODEV))
    # the needle calls: their own rules first, then the encoder or handle, then the report and radius
    valid = (NODEV, ENC_NODEV)
    add("locate_needle_damage_device", REPORT_RULES + LOCATE_RADIUS + [
        ("no-unowned", dict(unowned=False), BAD, UNOWNED),
        ("negative-records", dict(n_records=-1), BAD, RECORDS),
        ("no-records", dict(records=False), BAD, RECORDS),
        ("no-records-0", dict(records=False, n_records=0), *valid),
        ("no-unowned-no-records", dict(unowned=False, records=False), BAD, UNOWNED),
        ("no-records-no-encoder", dict(records=False, e=False), BAD, RECORDS),
        ("no-encoder", dict(e=False), BAD, NULL_ARG),
        ("no-shards", dict(shards=False), BAD, NULL_ARG),
        ("no-encoder-no-report", dict(e=False, report=False), BAD, NULL_ARG),
        ("bad-geometry", dict(dat_size=-1), BAD, "bad geometry"),
        ("bad-geometry-radius-3", dict(dat_size=-1, radius=3), BAD, R12),
        ("bad-geometry-null-shard", dict(dat_size=-1, null=(3,)), BAD, "bad geometry"),
        ("null-shard", dict(null=(3,)), BAD, "NULL shard"),
        ("valid", {}, *valid),
    ], valid)
    for call in ("ec_volume_locate_needle_damage", "ec_volume_repair_needle_damage"):
        valid = (NODEV, VOL_NODEV)
        rows = REPORT_RULES + LOCATE_RADIUS + [
            ("negative-needles-cap", dict(needles_cap=-1), BAD, NEEDLES),
            ("no-needles", dict(needles=False), BAD, NEEDLES),
            ("no-needles-cap-0", dict(needles=False, needles_cap=0), *valid),
            ("no-unowned", dict(unowned=False), BAD, UNOWNED),
            ("no-needles-no-unowned", dict(needles=False, unowned=False), BAD, NEEDLES),
            ("no-handle", dict(v=False), BAD, NULL_ARG),
            ("no-n-needles", dict(n_needles=False), BAD, NULL_ARG),
            ("no-ok", dict(ok=False), BAD, NULL_ARG),
            ("no-unowned-no-handle", dict(unowned=False, v=False), BAD, UNOWNED),
            ("no-handle-no-report", dict(v=False, report=False), BAD, NULL_ARG),
            ("no-handle-radius-3", dict(v=False, radius=3), BAD, NULL_ARG),
            ("valid", {}, *valid),
        ]
        if "repair" in call:
            rows += [
                ("no-checks", dict(checks=False), BAD, CHECKS),
                ("no-checks-cap-0", dict(checks=False, needles_cap=0), *valid),
                ("no-checks-no-unowned", dict(checks=False, unowned=False), BAD, UNOWNED),
                ("no-checks-no-handle", dict(checks=False, v=False), BAD, CHECKS),
                ("no-checks-radius-3", dict(checks=False, radius=3), BAD, CHECKS),
            ]
        add(call, rows, valid)
    # the sketch calls: pointers, shard_len, pages_cap, then the radius; the full-set call then 2·radius <= m and a
    # sketch per shard, the checked call the count of present sketches
    for call in ("locate_sketch_damage", "locate_sketch_damage_checked"):
        valid = (NODEV, ENC_NODEV)
        checked = call.endswith("checked")
        add(call, [
            ("no-encoder", dict(e=False), BAD, NULL_ARG),
            ("no-sketches", dict(sketches=False), BAD, NULL_ARG),
            ("no-n-flagged", dict(n_flagged=False), BAD, NULL_ARG),
            ("no-ok", dict(ok=False), BAD, NULL_ARG),
            ("negative-shard-len", dict(shard_len=-1), BAD, "shard_len must be >= 0"),
            ("negative-pages-cap", dict(pages_cap=-1), BAD, PAGES_CAP),
            ("no-pages", dict(pages=False), BAD, PAGES_CAP),
            ("no-pages-cap-0", dict(pages=False, pages_cap=0), *valid),
            ("radius-minus-1", dict(radius=-1), BAD, R012),
            ("radius-3", dict(radius=3), BAD, R012),
            ("radius-0", dict(radius=0), *valid),
            ("radius-2", dict(radius=2), *valid),
            ("radius-2-m-2", dict(radius=2, m=2), *(valid if checked else (BAD, parity(2, 2)))),
            ("radius-1-m-2", dict(radius=1, m=2), *valid),
            ("no-ok-negative-shard-len", dict(ok=False, shard_len=-1), BAD, NULL_ARG),
            ("negative-shard-len-no-pages", dict(shard_len=-1, pages=False), BAD, "shard_len must be >= 0"),
            ("no-pages-radius-3", dict(pages=False, radius=3), BAD, PAGES_CAP),
            ("lost", dict(lost=(4,)),
             *(valid if checked else (FEW, "no sketch of shard 4: rebuild it first"))),
            ("lost-radius-3", dict(lost=(4,), radius=3), BAD, R012),
            ("lost-radius-2-m-2", dict(lost=(1,), radius=2, m=2),
             *(valid if checked else (BAD, parity(2, 2)))),
            ("too-few", dict(lost=(0, 1, 2, 3, 4)),
             *((FEW, "fewer than data_shards sketches present") if checked
               else (FEW, "no sketch of shard 0: rebuild it first"))),
            ("too-few-radius-3", dict(lost=(0, 1, 2, 3, 4), radius=3), BAD, R012),
            ("valid", {}, *valid),
        ], valid)
    return out


CASES = cases()


@pytest.fixture(scope="module")
def env(swec, tmp_path_factory):
    e = Env(swec, tmp_path_factory.mktemp("rules"))
    yield e
    e.close()


@pytest.mark.parametrize("call,over,status,text", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_argument_rule(env, call, over, status, text):
    rc = CALLS[call](env, **over)
    got = (rc, env.L.swec_last_error().decode())
    assert got == (status, text.format(root=env.root))


def test_every_entry_point_is_covered():
    assert len(CALLS) == 14
    assert {c[1] for c in CASES} == set(CALLS)
