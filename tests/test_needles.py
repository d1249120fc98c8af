"""The needle check: Needle.ReadBytes (size, layout, CRC32-C) on the GPU, alone (swec_check_needles_device) and as the
needle parse of EcVolume.ScrubLocal (swec_ec_volume_scrub_needles)."""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import needle_oracle as no  # noqa: E402

from oracle import rs_numpy as rn  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_IDX = os.path.join(ROOT, "tests", "golden", "fixtures", "1.idx")
REF_DAT = os.path.join(ROOT, "oracle", "_ref", "1.dat")
MIB, GIB = 1 << 20, 1 << 30
SEED = 0x5EEDC4C3
OK, SIZE_MISMATCH, OUT_OF_RANGE, BAD_CRC, OUTSIDE = 0, 1, 2, 3, 4


def error_text(r) -> str | None:
    """The reference's wording of a device result (what the volume scrub reports after "needle <id> on volume <v>: ")."""
    if r["status"] == OK:
        return None
    if r["status"] == SIZE_MISMATCH:
        return "size mismatch"
    if r["status"] == OUT_OF_RANGE:
        return f"index out of range {r['range_index']}: needle data corrupted"
    if r["status"] == BAD_CRC:
        return (f"invalid CRC for needle {r['needle_id']:x} (got {r['crc_got']:08x}, want {r['crc_want']:08x}), "
                "data on disk corrupted: needle data corrupted")
    return "outside the image"


def ref_records():
    idx = open(REF_IDX, "rb").read()
    return [(k, o * 8, s) for k, o, s in rn._entries(idx) if s > 0]


# ------------------------------------------------------------------------------------------ CPU


def test_crc32c_check_value_and_host_agree():
    assert no.crc32c(b"123456789") == 0xE3069283
    assert no.host_crc32c(b"123456789") == 0xE3069283
    rng = np.random.default_rng(5)
    buf = rng.integers(0, 256, 1 << 16, dtype=np.uint8)
    offs, lens = [], []
    for _ in range(40):
        off, n = int(rng.integers(0, 4096)), int(rng.integers(0, 3000))
        assert no.crc32c(buf[off:off + n]) == no.host_crc32c(buf[off:off + n].copy())
        offs.append(off)
        lens.append(n)
    got = no.ranges_crc32c(buf, offs, lens, threads=3)
    assert [int(x) for x in got] == [no.crc32c(buf[o:o + n]) for o, n in zip(offs, lens)]


def test_synth_crc_matches_the_stream(oracle):
    offs, lens = [0, 8, 13, 100_003, 65_530], [0, 1, 70_001, 5, 200_000]
    got = no.synth_crc32c(SEED, offs, lens, threads=2)
    stream = oracle.synth(0, 300_000, SEED)
    assert [int(x) for x in got] == [no.crc32c(stream[o:o + n]) for o, n in zip(offs, lens)]


def test_read_bytes_restatement_wording():
    data = bytes(range(200))
    for v in (1, 2, 3):
        rec = no.write_record(0xABC, data, version=v)
        size = int.from_bytes(rec[12:16], "big")
        assert no.read_bytes(rec, size, v) is None
        assert no.read_bytes(rec, size + 1, v) == "size mismatch"
        bad = bytearray(rec)
        bad[16 + (4 if v > 1 else 0) + 7] ^= 1
        want = int.from_bytes(rec[16 + size:20 + size], "big")
        got = no.crc32c(bytes(bad[16 + (4 if v > 1 else 0):][:200]))
        assert no.read_bytes(bad, size, v) == (f"invalid CRC for needle abc (got {got:08x}, want {want:08x}), "
                                               "data on disk corrupted: needle data corrupted")
    rec = no.write_record(7, data, version=3, name=b"file.txt", mime=b"text/plain", last_modified=123, ttl=b"\x01\x02",
                          pairs=b'{"a":"b"}')
    size = int.from_bytes(rec[12:16], "big")
    assert no.read_bytes(rec, size, 3) is None
    cases = {1: 16, 2: 16 + 4 + 200 + 1}          # DataSize, name length
    for which, at in cases.items():
        bad = bytearray(rec)
        if which == 1:
            bad[at:at + 4] = (size).to_bytes(4, "big")
        else:
            bad[at] = 255
        assert no.read_bytes(bad, size, 3) == f"index out of range {which}: needle data corrupted"
    assert no.read_bytes(no.write_record(9, b"", version=3), 6, 3) == "size mismatch"
    assert no.read_bytes(no.write_record(9, b"", version=2, checksum=0x1234), 5, 2) is None   # no Data: no CRC
    # a body of 1..3 bytes cannot hold DataSize
    tiny = bytearray(no.write_record(9, b"", version=2))
    tiny[12:16] = (2).to_bytes(4, "big")
    assert no.read_bytes(tiny, 2, 2) == "index out of range 1: needle data corrupted"


@pytest.mark.skipif(not os.path.exists(REF_DAT), reason="oracle/_ref/1.dat not built")
def test_reference_fixture_fails_its_own_crc_check():
    """Every record of the reference's 1.dat stores CRC.Value() of its Data, not the raw CRC that ReadBytes compares."""
    dat = np.fromfile(REF_DAT, dtype=np.uint8)
    recs = ref_records()
    assert len(recs) == 298 and dat[0] == 3
    for k, off, size in recs:
        rec = dat[off:off + no.actual_size(size, 3)].tobytes()
        err, d_off, n = no.layout(rec, size, 3)
        got, want = no.crc32c(rec[d_off:d_off + n]), int.from_bytes(rec[16 + size:20 + size], "big")
        assert err is None and n > 0 and got != want and no.legacy_value(got) == want
        assert no.read_bytes(rec, size, 3).startswith(f"invalid CRC for needle {k:x} (got {got:08x}, want {want:08x})")


def test_needle_check_struct_matches_the_header(swec, tmp_path):
    from seaweedfs_b200._native import NeedleCheck
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "swec.h"\nint main(void){printf("%zu %zu %zu %zu %zu\\n",'
                   ' sizeof(swec_needle_check), offsetof(swec_needle_check, status), offsetof(swec_needle_check, crc_got),'
                   ' offsetof(swec_needle_check, legacy_crc), offsetof(swec_needle_check, reserved));return 0;}\n')
    exe = str(tmp_path / "s")
    subprocess.run(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", exe, str(src)], check=True)
    got = [int(x) for x in subprocess.run([exe], check=True, stdout=subprocess.PIPE, text=True).stdout.split()]
    assert got == [C.sizeof(NeedleCheck), NeedleCheck.status.offset, NeedleCheck.crc_got.offset,
                   NeedleCheck.legacy_crc.offset, NeedleCheck.reserved.offset]


def mounted_volume(oracle, tmp_path, seed=71, records=400, big=0, version=3, name="7"):
    """A miniature volume of well-formed records (some with every optional field), laid down as EC shards by the
    oracle with production block sizes.  Returns (base, dat, entries [(id, offset, size)])."""
    rng = np.random.default_rng(seed)
    dat = bytearray([version, 0, 0, 0, 0, 0, 0, 0])
    idx, entries = b"", []
    for i in range(records):
        n = big if (big and i == records // 2) else int(math.exp(rng.uniform(0, math.log(200_000)))) if rng.random() > 0.1 else 0
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        extra = {}
        if version > 1 and rng.random() < 0.4:
            extra = dict(name=b"n%d.bin" % i, mime=b"application/octet-stream", last_modified=1_700_000_000 + i,
                         ttl=b"\x03\x01", pairs=b'{"k":"%d"}' % i)
        rec = no.write_record(1000 + i, data, version=version, append_at_ns=i, **extra)
        size = int.from_bytes(rec[12:16], "big")
        entries.append((1000 + i, len(dat), size))
        idx += rn._entry(1000 + i, len(dat) // 8, size)
        dat += rec
    dat = np.frombuffer(bytes(dat), dtype=np.uint8).copy()
    base = str(tmp_path / name)
    for i, s in enumerate(oracle.encode_dat_image(dat)):
        s.tofile(base + ".ec%02d" % i)
    open(base + ".ecx", "wb").write(rn.sorted_ecx_from_idx(idx))
    json.dump({"version": version, "datFileSize": str(len(dat)), "ecShardConfig": {"dataShards": 10, "parityShards": 4}},
              open(base + ".vif", "w"))
    return base, dat, entries


def test_scrub_needles_without_a_device_fails(swec, oracle, tmp_path):
    ec = swec.erasure_coding
    base, _, entries = mounted_volume(oracle, tmp_path, records=20)
    vol = ec.EcVolume(base, device=-1)
    assert vol.scrub_local() == (len(entries), [], [])          # the walk alone needs no GPU
    with pytest.raises(swec._native.SwecError) as e:
        vol.scrub_needles(7)
    assert e.value.status == -7
    vol.close()


# ------------------------------------------------------------------------------------------ GPU


def shard_position(x, k=10, small=MIB):
    """Shard id and offset of .dat byte x in a volume with no large rows (< 10 GiB)."""
    row, col = divmod(x, k * small)
    return col // small, row * small + col % small


def poke_shard(base, x, value):
    sid, off = shard_position(x)
    with open(base + ".ec%02d" % sid, "r+b") as f:
        f.seek(off)
        f.write(bytes([value]))


def record_shards(off, n):
    return {shard_position(x)[0] for x in range(off - off % MIB, off + n, MIB)} | {shard_position(off + n - 1)[0]}


def expected_findings(dat, entries, vid, version=3, skip=lambda off, n: False):
    out = []
    for k, off, size in entries:
        n = no.actual_size(size, version)
        if skip(off, n):
            continue
        err = no.read_bytes(dat[off:off + n].tobytes(), size, version,
                            crc_of_data=lambda o, ln: no.host_crc32c(dat[off + o:off + o + ln].copy()))
        if err:
            out.append(f"needle {k} on volume {vid}: {err}")
    return out


def corrupt(base, dat, entries, rng, version=3):
    """One record of each kind: a flipped Data byte, a wrong header Size, a DataSize past the body, a name length past
    the body.  Written into the shard files and mirrored into `dat`."""
    with_data = [e for e in entries if e[2] > 40 and int.from_bytes(dat[e[1] + 16:e[1] + 20].tobytes(), "big") > 0]
    picks = rng.choice(len(with_data), 4, replace=False)
    done = []
    for kind, p in zip(("data", "size", "datasize", "name"), picks):
        k, off, size = with_data[int(p)]
        if kind == "data":
            x = off + 20 + int(rng.integers(0, int.from_bytes(dat[off + 16:off + 20].tobytes(), "big")))
            val = dat[x] ^ 0x40
        elif kind == "size":
            x, val = off + 15, dat[off + 15] ^ 0x08
        elif kind == "datasize":
            x, val = off + 16, 0x7F
        else:
            flags_at = off + 20 + int.from_bytes(dat[off + 16:off + 20].tobytes(), "big")
            if not dat[flags_at] & no.FLAG_NAME:
                continue
            x, val = flags_at + 1, 255
        dat[x] = val
        poke_shard(base, x, val)
        done.append(k)
    return done


@pytest.mark.gpu
def test_scrub_needles_on_a_mounted_volume(cuda, swec, oracle, tmp_path):
    ec = swec.erasure_coding
    vid = 7
    base, dat, entries = mounted_volume(oracle, tmp_path, seed=72, records=300)
    assert any(off // MIB != (off + no.actual_size(s, 3) - 1) // MIB for _, off, s in entries)   # records straddle blocks
    vol = ec.EcVolume(base, device=0)
    assert vol.scrub_needles(vid) == (len(entries), [], []) == vol.scrub_local()
    vol.close()

    rng = np.random.default_rng(9)
    bad_ids = corrupt(base, dat, entries, rng)
    assert len(bad_ids) >= 3
    want = expected_findings(dat, entries, vid)
    assert len(want) == len(bad_ids) and all(f" {k} on volume" in w for k, w in zip(sorted(bad_ids), sorted(want)))
    vol = ec.EcVolume(base, device=0)
    count, broken, findings = vol.scrub_needles(vid)
    assert (count, broken) == (len(entries), []) and findings == want
    assert vol.scrub_local() == (len(entries), [], [])
    vol.close()

    # a shard that is not local: records with chunks on it are skipped, the rest still checked
    os.rename(base + ".ec03", base + ".ec03.away")
    vol = ec.EcVolume(base, device=0)
    count, broken, findings = vol.scrub_needles(vid)
    assert findings == expected_findings(dat, entries, vid, skip=lambda off, n: 3 in record_shards(off, n))
    assert (count, broken) == (len(entries), []) and vol.scrub_local()[2] == []
    vol.close()
    os.rename(base + ".ec03.away", base + ".ec03")

    # a truncated shard: scrub_local's findings, needle findings of the records walked before the stop, then the stop
    os.truncate(base + ".ec00", os.path.getsize(base + ".ec00") // 2)
    vol = ec.EcVolume(base, device=0)
    local = vol.scrub_local()
    count, broken, findings = vol.scrub_needles(vid)
    assert (count, broken) == local[:2] and [f for f in findings if not f.startswith("needle ")] == local[2]
    assert findings[-1] == local[2][-1] and local[2][-1].startswith("expected ")
    walked = sorted(entries, key=lambda e: e[0])[:count]
    stop = walked[-1][0]
    want = expected_findings(dat, walked[:-1], vid)
    assert [f for f in findings if f.startswith("needle ")] == want, stop
    vol.close()


@pytest.mark.gpu
def test_scrub_needles_checks_a_record_larger_than_a_slot(cuda, swec, oracle, tmp_path):
    ec = swec.erasure_coding
    base, dat, entries = mounted_volume(oracle, tmp_path, seed=73, records=12, big=66 * MIB + 12345)
    big = max(entries, key=lambda e: e[2])
    vol = ec.EcVolume(base, device=0)
    assert vol.scrub_needles(3) == (len(entries), [], [])
    vol.close()
    x = big[1] + 20 + 66 * MIB     # late in the record's Data
    dat[x] ^= 1
    poke_shard(base, x, int(dat[x]))
    vol = ec.EcVolume(base, device=0)
    count, broken, findings = vol.scrub_needles(3)
    assert findings == expected_findings(dat, entries, 3) and len(findings) == 1
    assert findings[0].startswith(f"needle {big[0]} on volume 3: invalid CRC for needle {big[0]:x} (got ")
    vol.close()


@pytest.mark.gpu
@pytest.mark.skipif(not os.path.exists(REF_DAT), reason="oracle/_ref/1.dat not built")
def test_reference_fixture_on_the_gpu(cuda, swec):
    torch = cuda
    ec = swec.erasure_coding
    dat = np.fromfile(REF_DAT, dtype=np.uint8)
    recs = ref_records()
    d = torch.from_numpy(dat).cuda()
    out = ec.check_needles_device(d.data_ptr(), len(dat), recs, needle_version=3, device=0)
    for (k, off, size), r in zip(recs, out):
        rec = dat[off:off + no.actual_size(size, 3)].tobytes()
        _, d_off, n = no.layout(rec, size, 3)
        got = no.crc32c(rec[d_off:d_off + n])
        assert (r["status"], r["crc_got"], r["data_size"], r["legacy_crc"]) == (BAD_CRC, got, n, 1), k
        assert r["crc_want"] == no.legacy_value(got)
        assert f"needle {k}: {error_text(r)}" == f"needle {k}: {no.read_bytes(rec, size, 3)}"
    # entries past the image's end are never read
    out = ec.check_needles_device(d.data_ptr(), len(dat), [(1, len(dat) - 16, 100), (2, -8, 0), (3, len(dat), 0)],
                                  needle_version=3, device=0)
    assert [r["status"] for r in out] == [OUTSIDE] * 3
    assert ec.check_needles_device(d.data_ptr(), len(dat), [], device=0) == []


def synthetic_image(version, total, big, rng):
    """A seeded record set over `total` bytes of the synthetic stream: sizes log-uniform from 1 B to 8 MiB, some empty,
    some of 1-64 B, a fraction with name / mime / TTL / pairs, and one record of `big` bytes.  Returns the records
    (id, offset, size, data offset, data length) and the header / tail bytes to write over the stream."""
    recs, patches = [], []
    pos, i = 8, 0
    lengths, extras = [], []
    while True:
        r = rng.random()
        n = big if i == 1 else 0 if r < 0.03 else int(rng.integers(1, 65)) if r < 0.1 else \
            int(math.exp(rng.uniform(0, math.log(8 * MIB))))
        extra = {}
        if version > 1 and rng.random() < 0.25:
            extra = dict(name=b"name-%d" % i, mime=b"image/png" if i % 2 else b"", last_modified=1_600_000_000 + i,
                         ttl=b"\x05\x03" if i % 3 else None, pairs=b'{"x":%d}' % i if i % 5 else None)
        head = 16 + (4 if version > 1 else 0)
        tail_fields = len(no.body(b"", **extra)) - 4 if version > 1 else 0
        size = (4 if version > 1 else 0) + n + tail_fields
        span = no.actual_size(size, version)
        if pos + span > total:
            break
        recs.append((10_000 + i, pos, size, pos + head, n))
        extras.append(extra)
        lengths.append(n)
        pos += span
        i += 1
    return recs, extras


def lay_records(torch, img, version, recs, extras, crcs):
    idx, vals = [], []
    for (k, off, size, d_off, n), extra, crc in zip(recs, extras, crcs):
        head = (0x0BADF00D).to_bytes(4, "big") + k.to_bytes(8, "big") + size.to_bytes(4, "big")
        if version > 1:
            head += n.to_bytes(4, "big")
            tail = no.body(b"", **extra)[4:]
        else:
            tail = b""
        tail += int(crc).to_bytes(4, "big") + ((k * 7919).to_bytes(8, "big") if version == 3 else b"")
        tail += bytes(no.actual_size(size, version) - (d_off - off) - n - len(tail))
        idx.append(np.arange(off, off + len(head), dtype=np.int64))
        vals.append(np.frombuffer(head, dtype=np.uint8))
        idx.append(np.arange(d_off + n, d_off + n + len(tail), dtype=np.int64))
        vals.append(np.frombuffer(tail, dtype=np.uint8))
    i = torch.from_numpy(np.concatenate(idx)).cuda()
    v = torch.from_numpy(np.concatenate(vals)).cuda()
    img[i] = v
    del i, v


def check_image(torch, swec, img, size, version, recs, extras, crcs, rng):
    ec = swec.erasure_coding
    entries = [(k, off, s) for k, off, s, _, _ in recs]
    out = ec.check_needles_device(img.data_ptr(), size, entries, needle_version=version, device=0)
    bad = [(r["needle_id"], r["status"]) for r in out if r["status"] != OK]
    assert bad == []
    for (k, off, s, d_off, n), crc, r in zip(recs, crcs, out):
        assert r["data_size"] == n and r["crc_want"] == crc and (n == 0 or r["crc_got"] == crc), k

    # damage: a Data byte, a header Size, a DataSize, a name length
    small = [j for j, rec in enumerate(recs) if 16 < rec[4] <= 8 * MIB]
    named = [j for j, e in enumerate(extras) if e.get("name")]
    picks = rng.choice(small, 8, replace=False)
    damaged = {}
    for j in picks[:4]:
        k, off, s, d_off, n = recs[j]
        x = d_off + int(rng.integers(0, n))
        img[x] ^= 0x21
        damaged[j] = None
    for j in picks[4:6]:
        k, off, s, d_off, n = recs[j]
        img[off + 14] ^= 0x01
        damaged[j] = None
    if version > 1:
        for j in picks[6:8]:
            k, off, s, d_off, n = recs[j]
            img[off + 16:off + 20] = torch.tensor([0, 0xFF, 0xFF, 0xFF], dtype=torch.uint8, device=img.device)
            damaged[j] = None
        for j in rng.choice(named, 2, replace=False):
            k, off, s, d_off, n = recs[j]
            img[d_off + n + 1] = 255
            damaged[j] = None
    torch.cuda.synchronize()
    out = ec.check_needles_device(img.data_ptr(), size, entries, needle_version=version, device=0)
    flagged = {j for j, r in enumerate(out) if r["status"] != OK}
    assert flagged == set(damaged)
    for j in damaged:
        k, off, s, d_off, n = recs[j]
        rec = img[off:off + no.actual_size(s, version)].cpu().numpy()
        want = no.read_bytes(rec.tobytes(), s, version, crc_of_data=lambda o, ln: no.host_crc32c(rec[o:o + ln].copy()))
        assert error_text(out[j]) == want, (k, out[j])
        if out[j]["status"] == BAD_CRC:
            assert out[j]["crc_got"] == no.host_crc32c(rec[d_off - off:d_off - off + n].copy()) and not out[j]["legacy_crc"]


@pytest.mark.gpu
@pytest.mark.parametrize("version,size,big", [(3, 30 * GIB, 1536 * MIB), (2, 3 * GIB, 300 * MIB), (1, 3 * GIB, 300 * MIB)])
def test_check_needles_device_full_size(cuda, swec, version, size, big):
    """A volume image in HBM filled from the seeded stream, needle headers and tails written over it: every record
    checks OK with the oracle's CRC; exactly the damaged records are flagged, with the oracle's verdict."""
    torch = cuda
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < size + (4 << 30):
        pytest.skip(f"needs {size + (4 << 30)} B of free HBM, {free} free")
    rng = np.random.default_rng(1000 + version)
    recs, extras = synthetic_image(version, size, big, rng)
    assert len(recs) > 1000 and any(r[4] == 0 for r in recs) and any(r[4] == big for r in recs)
    crcs = no.synth_crc32c(SEED, [r[3] for r in recs], [r[4] for r in recs])
    img = torch.empty(size, dtype=torch.uint8, device="cuda")
    L = swec.lib()
    swec._native.check(L.swec_synth_fill_device(0, img.data_ptr(), 0, size, SEED, None))
    torch.cuda.synchronize()
    img[0] = version
    lay_records(torch, img, version, recs, extras, crcs)
    torch.cuda.synchronize()
    try:
        check_image(torch, swec, img, size, version, recs, extras, crcs, rng)
    finally:
        del img
        torch.cuda.empty_cache()
