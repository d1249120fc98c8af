"""Checker for the GPU needle check (tests and benchmarks only; the product never imports it).

- crc32c: CRC32-C (Castagnoli) as Go's crc32.Update(0, crc32.MakeTable(crc32.Castagnoli), data), restated in Python.
- write_record: a needle record of version 1, 2 or 3 with any of the optional fields (needle_write_v*.go layout).
- read_bytes: Needle.ReadBytes(record, 0, size, version) restated (needle_read.go:59-190, needle_read_tail.go:11-34):
  the reference's error text, or None.
- host(): the C CRC32-C (tests/c/crc32c_oracle.c), compiled into a temporary directory on first use, for bulk data.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

_TABLE = []
for _i in range(256):
    _c = _i
    for _ in range(8):
        _c = (_c >> 1) ^ 0x82F63B78 if _c & 1 else _c >> 1
    _TABLE.append(_c)
TABLE = np.array(_TABLE, dtype=np.uint32)

FLAG_NAME, FLAG_MIME, FLAG_LAST_MODIFIED, FLAG_TTL, FLAG_PAIRS = 0x02, 0x04, 0x08, 0x10, 0x20


def crc32c(data, crc: int = 0) -> int:
    c = crc ^ 0xFFFFFFFF
    for b in bytes(data):
        c = _TABLE[(c ^ b) & 0xFF] ^ (c >> 8)
    return c ^ 0xFFFFFFFF


def legacy_value(c: int) -> int:
    """CRC.Value() (crc.go:25-27): the form checksums were stored in before SeaweedFS 3.09."""
    return (((c >> 15) | (c << 17)) + 0xA282EAD8) & 0xFFFFFFFF


def actual_size(size: int, version: int) -> int:
    fixed = 16 + size + 4 + (8 if version == 3 else 0)
    return fixed + (8 - fixed % 8)


def body(data: bytes, name: bytes = b"", mime: bytes = b"", last_modified: int | None = None,
         ttl: bytes | None = None, pairs: bytes | None = None) -> bytes:
    """The v2/v3 body: DataSize, Data, Flags and the optional fields in the order readNeedleDataVersion2 reads them."""
    flags = (FLAG_NAME if name else 0) | (FLAG_MIME if mime else 0) | \
        (FLAG_LAST_MODIFIED if last_modified is not None else 0) | (FLAG_TTL if ttl is not None else 0) | \
        (FLAG_PAIRS if pairs is not None else 0)
    out = bytearray(len(data).to_bytes(4, "big") + bytes(data) + bytes([flags]))
    if name:
        out += bytes([len(name)]) + name
    if mime:
        out += bytes([len(mime)]) + mime
    if last_modified is not None:
        out += last_modified.to_bytes(5, "big")
    if ttl is not None:
        out += ttl
    if pairs is not None:
        out += len(pairs).to_bytes(2, "big") + pairs
    return bytes(out)


def write_record(needle_id: int, data: bytes, version: int = 3, cookie: int = 0x1234ABCD, checksum: int | None = None,
                 append_at_ns: int = 0, **fields) -> bytes:
    """A whole record: header, body (v1: Data alone), checksum, v3 timestamp, padding to 8."""
    b = bytes(data) if version == 1 else body(data, **fields)
    size = len(b)
    crc = crc32c(data) if checksum is None else checksum
    rec = cookie.to_bytes(4, "big") + needle_id.to_bytes(8, "big") + size.to_bytes(4, "big") + b + crc.to_bytes(4, "big")
    if version == 3:
        rec += append_at_ns.to_bytes(8, "big")
    return rec + bytes(actual_size(size, version) - len(rec))


def layout(rec, size: int, version: int):
    """ReadBytes up to the CRC: ("size mismatch" | "index out of range N" | None, data offset, data size)."""
    rec = bytes(rec)
    if int.from_bytes(rec[12:16], "big", signed=True) != size or size < 0:
        return "size mismatch", 16, 0
    if version == 1:
        return None, 16, size
    b, n, i = rec[16:16 + size], size, 0
    d_off, d_size = 16, 0
    if i < n:
        ds = int.from_bytes(rec[16:20], "big")   # a body of 1..3 bytes reads into the checksum, as Go's slice does
        i += 4
        if ds + i > n:
            return "index out of range 1", 16, 0
        d_off, d_size = 20, ds
        i += ds
    flags = 0
    if i < n:
        flags = b[i]
        i += 1
    if i < n and flags & FLAG_NAME:
        ln = b[i]
        i += 1
        if ln + i > n:
            return "index out of range 2", 16, 0
        i += ln
    if i < n and flags & FLAG_MIME:
        ln = b[i]
        i += 1
        if ln + i > n:
            return "index out of range 3", 16, 0
        i += ln
    if i < n and flags & FLAG_LAST_MODIFIED:
        if 5 + i > n:
            return "index out of range 4", 16, 0
        i += 5
    if i < n and flags & FLAG_TTL:
        if 2 + i > n:
            return "index out of range 5", 16, 0
        i += 2
    if i < n and flags & FLAG_PAIRS:
        if 2 + i > n:
            return "index out of range 6", 16, 0
        ln = int.from_bytes(b[i:i + 2], "big")
        i += 2
        if ln + i > n:
            return "index out of range 7", 16, 0
    return None, d_off, d_size


def read_bytes(rec, size: int, version: int, crc_of_data=None) -> str | None:
    """Needle.ReadBytes(rec, 0, size, version)'s error text, or None.  crc_of_data(offset, length) may supply the
    CRC of Data for records too large to checksum in Python."""
    rec = bytes(rec)
    err, off, n = layout(rec, size, version)
    if err == "size mismatch":
        return err
    if err:
        return err + ": needle data corrupted"
    if n == 0:
        return None
    got = crc_of_data(off, n) if crc_of_data else crc32c(rec[off:off + n])
    want = int.from_bytes(rec[16 + size:20 + size], "big")
    if got != want:
        nid = int.from_bytes(rec[4:12], "big")
        return (f"invalid CRC for needle {nid:x} (got {got:08x}, want {want:08x}), data on disk corrupted: "
                "needle data corrupted")
    return None


# ------------------------------------------------------------------ the C CRC32-C

_host = None


def host() -> C.CDLL:
    global _host
    if _host is None:
        out = os.path.join(tempfile.mkdtemp(prefix="crc32c_oracle_"), "libcrc32c_oracle.so")
        subprocess.run(["cc", "-O3", "-std=gnu11", "-fPIC", "-shared", "-pthread", "-o", out,
                        os.path.join(HERE, "c", "crc32c_oracle.c")], check=True)
        L = C.CDLL(out)
        L.orc_crc32c_update.restype = C.c_uint32
        L.orc_crc32c_update.argtypes = [C.c_uint32, C.c_void_p, C.c_size_t]
        L.orc_crc32c_ranges.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.orc_synth_crc32c.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        _host = L
    return _host


def host_crc32c(data) -> int:
    a = np.ascontiguousarray(np.frombuffer(bytes(data), dtype=np.uint8) if not isinstance(data, np.ndarray) else data)
    return int(host().orc_crc32c_update(0, a.ctypes.data, a.nbytes))


def ranges_crc32c(base: np.ndarray, offsets, lengths, threads: int | None = None) -> np.ndarray:
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    ln = np.ascontiguousarray(lengths, dtype=np.int64)
    out = np.zeros(len(off), dtype=np.uint32)
    host().orc_crc32c_ranges(base.ctypes.data, off.ctypes.data, ln.ctypes.data, out.ctypes.data, len(off),
                             threads or os.cpu_count() or 1)
    return out


def synth_crc32c(seed: int, offsets, lengths, threads: int | None = None) -> np.ndarray:
    """CRC32-C of byte ranges of the synthetic stream swec_synth_fill_device writes, never held in memory."""
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    ln = np.ascontiguousarray(lengths, dtype=np.int64)
    out = np.zeros(len(off), dtype=np.uint32)
    host().orc_synth_crc32c(seed, off.ctypes.data, ln.ctypes.data, out.ctypes.data, len(off),
                            threads or os.cpu_count() or 1)
    return out
