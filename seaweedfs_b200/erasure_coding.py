"""Host-side mirror of SeaweedFS's ``weed/storage/erasure_coding`` package surface for the RS hot
path, bound to libswec.so.  Names follow the Go package (Go spelling kept as aliases) so the parity
tests read like the reference's own tests:

    ECContext / NewDefaultECContext / CreateEncoder       ec_context.go:11-46
    Encoder.Encode / Reconstruct / ReconstructData        klauspost Encoder, call sites
                                                          ec_encoder.go:265,360; store_ec.go:551
    WriteEcFiles / generateEcFiles / RebuildEcFiles       ec_encoder.go:61-128,146-200
    WriteDatFile                                          ec_decoder.go:176-223
    LocateData / Interval.ToShardIdAndOffset              ec_locate.go:16-98

Buffers are numpy uint8 arrays (host) or raw device pointers (ints) for the ``*_device`` calls.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from ._native import (STATUS, DamageRange, DamageReport, Interval, NeedleDamage, NeedleRead, ReconstructItem, SketchPage,
                      SwecError, check, lib)

DataShardsCount = 10                               # ec_encoder.go:20
ParityShardsCount = 4                              # ec_encoder.go:21
TotalShardsCount = DataShardsCount + ParityShardsCount
MaxShardCount = 32                                 # ec_encoder.go:23
ErasureCodingLargeBlockSize = 1024 * 1024 * 1024   # ec_encoder.go:25
ErasureCodingSmallBlockSize = 1024 * 1024          # ec_encoder.go:26


def _ptrs(arrs) -> C.Array:
    out = (C.c_void_p * len(arrs))()
    for i, a in enumerate(arrs):
        if a is None:
            out[i] = None
        elif isinstance(a, np.ndarray):
            out[i] = a.ctypes.data
        else:
            out[i] = int(a)
    return out


def _fill_missing(shards: list, n: int, data_shards: int, data_only: bool, need_data_shards: bool = True):
    """The presence mask of a reconstruct call's shards, with the shards it rebuilds put in place as new zeroed
    arrays, and the pointer list it takes (NULL for a shard that stays missing)."""
    present = np.array([s is not None and len(s) > 0 for s in shards], dtype=np.uint8)
    if need_data_shards and present.sum() < data_shards:
        raise SwecError(-2, "too few shards given (ErrTooFewShards)")
    for i in range(len(shards)):
        if not present[i] and (i < data_shards or not data_only):
            shards[i] = np.zeros(n, dtype=np.uint8)
    return present, _ptrs([s if s is not None and len(s) else None for s in shards])


class Encoder:
    """reedsolomon.Encoder backed by the GPU engine (swec_encoder)."""

    def __init__(self, data_shards: int, parity_shards: int, device: int = 0):
        h = C.c_void_p()
        check(lib().swec_encoder_new(data_shards, parity_shards, device, C.byref(h)))
        self._h = h
        self.data_shards, self.parity_shards, self.device = data_shards, parity_shards, device

    def close(self) -> None:
        h, self._h = getattr(self, "_h", None), None
        if h and callable(lib):        # module globals are already cleared when this runs at interpreter exit
            lib().swec_encoder_free(h)

    __del__ = close

    @property
    def total_shards(self) -> int:
        return self.data_shards + self.parity_shards

    def matrix(self) -> np.ndarray:
        m = np.zeros((self.total_shards, self.data_shards), dtype=np.uint8)
        check(lib().swec_encoder_matrix(self._h, m.ctypes.data))
        return m

    def reconstruct_matrix(self, present, data_only: bool = False):
        pres = np.ascontiguousarray(np.asarray(present, dtype=np.uint8))
        inputs = (C.c_int * self.data_shards)()
        outputs = (C.c_int * self.total_shards)()
        n = C.c_int(0)
        rows = np.zeros((self.total_shards, self.data_shards), dtype=np.uint8)
        check(lib().swec_reconstruct_matrix(self._h, pres.ctypes.data, int(data_only), inputs, outputs,
                                            C.byref(n), rows.ctypes.data))
        return list(inputs), list(outputs[: n.value]), rows[: n.value].copy()

    # -- host buffers ---------------------------------------------------------------------------
    def _check_shards(self, shards, allow_missing: bool):
        if len(shards) != self.total_shards:
            raise SwecError(-1, f"need {self.total_shards} shards, got {len(shards)} (ErrTooFewShards)")
        n = None
        for s in shards:
            if s is None or (allow_missing and len(s) == 0):
                if not allow_missing:
                    raise SwecError(-1, "nil shard")
                continue
            if s.dtype != np.uint8 or not s.flags["C_CONTIGUOUS"]:
                raise SwecError(-1, "shards must be contiguous uint8 arrays")
            if n is None:
                n = s.shape[0]
            elif s.shape[0] != n:
                raise SwecError(-6, "shards are of different sizes (ErrShardSize)")
        if not n:
            raise SwecError(-1, "no shard data (ErrShardNoData)")
        return n

    def encode(self, shards: list[np.ndarray]) -> None:
        """Encode(shards [][]byte): parity slices (last m) are overwritten in place."""
        n = self._check_shards(shards, allow_missing=False)
        check(lib().swec_encode(self._h, _ptrs(shards), n))

    def reconstruct(self, shards: list, data_only: bool = False) -> None:
        """Reconstruct(shards): None / empty entries are missing and are replaced by new arrays."""
        n = self._check_shards(shards, allow_missing=True)
        present, ptrs = _fill_missing(shards, n, self.data_shards, data_only)
        check(lib().swec_reconstruct(self._h, ptrs, present.ctypes.data, n, int(data_only)))

    def reconstruct_data(self, shards: list) -> None:
        self.reconstruct(shards, data_only=True)

    def reconstruct_batch(self, batch: list[list], data_only: bool = True) -> None:
        """Many Reconstruct/ReconstructData calls in one crossing (batched degraded reads): each
        element is a shards list as for reconstruct(); missing entries are filled in place."""
        items = (ReconstructItem * len(batch))()
        keep = []
        for j, shards in enumerate(batch):
            n = self._check_shards(shards, allow_missing=True)
            present, ptrs = _fill_missing(shards, n, self.data_shards, data_only, need_data_shards=False)
            keep.append((ptrs, present))
            items[j].shards = C.cast(ptrs, C.POINTER(C.c_void_p))
            items[j].present = present.ctypes.data_as(C.POINTER(C.c_uint8))
            items[j].shard_len = n
            items[j].data_only = int(data_only)
        check(lib().swec_reconstruct_batch(self._h, items, len(batch)))

    def verify(self, shards: list[np.ndarray]) -> bool:
        n = self._check_shards(shards, allow_missing=False)
        ok = C.c_int(0)
        check(lib().swec_verify(self._h, _ptrs(shards), n, C.byref(ok)))
        return bool(ok.value)

    # -- device buffers (raw pointers), asynchronous on `stream` ----------------------------------
    def encode_device(self, data_ptrs, parity_ptrs, shard_len: int, stream: int = 0) -> None:
        check(lib().swec_encode_device(self._h, _ptrs(data_ptrs), _ptrs(parity_ptrs), shard_len, stream))

    def reconstruct_device(self, shard_ptrs, present, shard_len: int, data_only: bool = False, stream: int = 0) -> None:
        pres = np.ascontiguousarray(np.asarray(present, dtype=np.uint8))
        check(lib().swec_reconstruct_device(self._h, _ptrs(shard_ptrs), pres.ctypes.data, shard_len,
                                            int(data_only), stream))

    def apply_device(self, rows, in_ptrs, out_ptrs, shard_len: int, stream: int = 0) -> None:
        """out[p] = XOR_i rows[p][i] ⊗ in[i] for an arbitrary matrix (device pointers)."""
        rows = np.ascontiguousarray(rows, dtype=np.uint8)
        check(lib().swec_apply_device(self._h, rows.shape[0], rows.shape[1], rows.ctypes.data, _ptrs(in_ptrs),
                                      _ptrs(out_ptrs), shard_len, stream))

    def encode_volume_device(self, dat_ptr: int, dat_size: int, parity_ptrs, stream: int = 0,
                             large_block: int = ErasureCodingLargeBlockSize,
                             small_block: int = ErasureCodingSmallBlockSize) -> None:
        check(lib().swec_encode_volume_device(self._h, dat_ptr, dat_size, large_block, small_block,
                                              _ptrs(parity_ptrs), stream))

    def extract_data_shard_device(self, dat_ptr: int, dat_size: int, shard_id: int, out_ptr: int, stream: int = 0,
                                  large_block: int = ErasureCodingLargeBlockSize,
                                  small_block: int = ErasureCodingSmallBlockSize) -> None:
        check(lib().swec_extract_data_shard_device(self._h, dat_ptr, dat_size, large_block, small_block,
                                                   shard_id, out_ptr, stream))

    def write_dat_device(self, data_shard_ptrs, dat_size: int, dat_out_ptr: int, stream: int = 0,
                         large_block: int = ErasureCodingLargeBlockSize,
                         small_block: int = ErasureCodingSmallBlockSize) -> None:
        """WriteDatFile on device memory (ec_decoder.go:176-223): un-stripe the k data shards into the volume image."""
        check(lib().swec_write_dat_device(self._h, _ptrs(data_shard_ptrs), dat_size, large_block, small_block,
                                          dat_out_ptr, stream))

    def locate_damage_device(self, shard_ptrs, shard_len: int, radius: int = 1, max_ranges: int = 4096,
                             stream: int = 0) -> dict:
        """Which shards of k+m shards in device memory are wrong, from the parity syndrome of every byte column
        (swec_locate_damage_device).  Same result as locate_ec_damage, without "ok"."""
        out = _DamageOut(max_ranges)
        check(lib().swec_locate_damage_device(self._h, _ptrs(shard_ptrs), shard_len, radius, *out.args, stream))
        return out.result()

    def correct_damage_device(self, shard_ptrs, shard_len: int, radius: int = 1, max_ranges: int = 4096,
                              stream: int = 0) -> dict:
        """locate_damage_device, which also corrects the located bytes in place (swec_correct_damage_device).  Returns
        the report of the shards as they were; uncorrectable columns are left as they were.  Radius 2 can miscorrect a
        column with 3 or more wrong shards (include/swec.h)."""
        out = _DamageOut(max_ranges)
        check(lib().swec_correct_damage_device(self._h, _ptrs(shard_ptrs), shard_len, radius, *out.args, stream))
        return out.result()

    def locate_needle_damage_device(self, shard_ptrs, shard_len: int, dat_size: int, records, radius: int = 1,
                                    large_block: int = ErasureCodingLargeBlockSize,
                                    small_block: int = ErasureCodingSmallBlockSize, max_ranges: int = 4096,
                                    stream: int = 0) -> dict:
        """locate_damage_device, and which records of the volume image striped into the data shards the damage hits
        (swec_locate_needle_damage_device).  records: (needle_id, offset, size) of every live record, sized as needle
        version 3.  Returns the result of locate_damage_device plus "needles" (one dict per record, in order, zero counts
        included) and "unowned" = [damaged, uncorrectable] bytes that no record owns.  The shards are only read."""
        records = list(records)
        arr = (NeedleDamage * max(1, len(records)))()
        for r, (nid, off, size) in zip(arr, records):
            r.needle_id, r.offset, r.size = nid, off, size
        out, unowned = _DamageOut(max_ranges), (C.c_uint64 * 2)()
        check(lib().swec_locate_needle_damage_device(self._h, _ptrs(shard_ptrs), shard_len, dat_size, large_block,
                                                     small_block, radius, arr, len(records), *out.args, unowned, stream))
        return {**out.result(), "needles": _needle_damage(arr[:len(records)]),
                "unowned": [int(unowned[0]), int(unowned[1])]}

    def reconstruct_checked_device(self, shard_ptrs, present, shard_len: int, radius: int = 1, max_ranges: int = 4096,
                                   stream: int = 0) -> dict:
        """reconstruct_device that reads every present shard and corrects the damage it locates in the first k present
        before it reaches the rebuilt shards (swec_reconstruct_checked_device).  Present shards are only read.  Returns
        the report of locate_damage_device over the present shards; radius 0 only detects (include/swec.h)."""
        pres, out = np.ascontiguousarray(np.asarray(present, dtype=np.uint8)), _DamageOut(max_ranges)
        check(lib().swec_reconstruct_checked_device(self._h, _ptrs(shard_ptrs), pres.ctypes.data, shard_len, radius,
                                                    *out.args, stream))
        return out.result()

    def decode_data_checked_device(self, shard_ptrs, present, shard_len: int, radius: int = 1, max_ranges: int = 4096,
                                   stream: int = 0) -> dict:
        """reconstruct_checked_device for ec.decode (swec_decode_data_checked_device): the present data shards are
        corrected in place and the missing data shards rebuilt, from any k present shards; parity shards are only read
        and a missing one may be None.  Returns the report of reconstruct_checked_device for the same shards; radius 0
        only detects (include/swec.h)."""
        pres, out = np.ascontiguousarray(np.asarray(present, dtype=np.uint8)), _DamageOut(max_ranges)
        check(lib().swec_decode_data_checked_device(self._h, _ptrs(shard_ptrs), pres.ctypes.data, shard_len, radius,
                                                    *out.args, stream))
        return out.result()

    def heal_device(self, shard_ptrs, present, shard_len: int, radius: int = 1, max_ranges: int = 4096,
                    stream: int = 0) -> dict:
        """reconstruct_checked_device that also corrects the damage it locates in the present shards, in place
        (swec_heal_device): columns within the radius become the true codeword, uncorrectable ones keep their present
        bytes.  Returns the report of reconstruct_checked_device for the same shards (include/swec.h)."""
        pres, out = np.ascontiguousarray(np.asarray(present, dtype=np.uint8)), _DamageOut(max_ranges)
        check(lib().swec_heal_device(self._h, _ptrs(shard_ptrs), pres.ctypes.data, shard_len, radius, *out.args, stream))
        return out.result()

    def page_sketch_device(self, shard_ptr: int, shard_len: int, sketches_ptr: int, seed: int, first_column: int = 0,
                           stream: int = 0) -> None:
        """The page sketches (include/swec.h, SWEC_PAGE_SKETCH_VERSION) of shard_len bytes of one shard in device
        memory, whose first byte is shard offset first_column (a multiple of 4096), into ceil(shard_len / 4096) words
        at sketches_ptr on this encoder's device (swec_page_sketch_device).  Asynchronous on `stream`."""
        check(lib().swec_page_sketch_device(self.device, shard_ptr, shard_len, first_column, seed, sketches_ptr, stream))

    def locate_sketch_damage(self, sketches, shard_len, radius: int = 1) -> dict:
        """Which pages of which shards are damaged, from the k+m shards' page sketches, all taken with one seed
        (swec_locate_sketch_damage).  sketches: k+m uint64 arrays (None: a lost shard, SWEC_ERR_TOO_FEW_SHARDS).
        shard_len: the shard length, or the k+m lengths the holders reported, which must be equal (ErrShardSize).
        Returns ok, "pages" = [(page, blamed shard mask, uncorrectable)] in ascending page order, "n_flagged" and
        "shard_pages" = {shard id: pages blamed on it}.  The result is per page, not per column (include/swec.h)."""
        shard_len, n_pages, ptrs, _ = self._sketch_args(sketches, shard_len)
        pages = (SketchPage * max(1, n_pages))()
        n, per_shard, ok = C.c_int64(0), (C.c_uint64 * MaxShardCount)(), C.c_int(0)
        check(lib().swec_locate_sketch_damage(self._h, ptrs, shard_len, radius, pages, n_pages, C.byref(n), per_shard,
                                              C.byref(ok)))
        return _sketch_result(ok, n, pages, per_shard)

    def locate_sketch_damage_checked(self, sketches, shard_len, radius: int = 1) -> dict:
        """locate_sketch_damage for a set with lost shards (swec_locate_sketch_damage_checked): None marks a lost shard,
        and the first k present shards are checked against the other c present ones at radius min(radius, c // 2).
        shard_len: as for locate_sketch_damage, the lengths the present shards' holders reported (None entries are
        skipped).  Returns the keys of locate_sketch_damage, plus "checks" = c and "rebuilt" = {lost shard id: uint64
        array}, the sketch that shard must have once rebuilt: of the true shard outside uncorrectable pages, and of what
        the plain rebuild writes on them.  With c = 0 nothing is checked and "ok" is False (include/swec.h)."""
        if not isinstance(shard_len, int):
            shard_len = [n for n in shard_len if n is not None]
        shard_len, n_pages, ptrs, keep = self._sketch_args(sketches, shard_len)
        present = sum(s is not None for s in keep)
        rebuilt = {i: np.zeros(n_pages, dtype=np.uint64) for i, s in enumerate(keep) if s is None}
        outs = (C.c_void_p * self.total_shards)(*[rebuilt[i].ctypes.data if i in rebuilt else None
                                                  for i in range(self.total_shards)])
        pages = (SketchPage * max(1, n_pages))()
        n, per_shard, ok = C.c_int64(0), (C.c_uint64 * MaxShardCount)(), C.c_int(0)
        check(lib().swec_locate_sketch_damage_checked(self._h, ptrs, shard_len, radius, pages, n_pages, C.byref(n),
                                                      per_shard, outs, C.byref(ok)))
        res = _sketch_result(ok, n, pages, per_shard)
        res["checks"] = max(0, present - self.data_shards)
        res["rebuilt"] = rebuilt
        return res

    def _sketch_args(self, sketches, shard_len):
        """(shard_len, pages, pointer array, arrays kept alive) of the sketch calls; shard_len may be a list of equal
        lengths (ErrShardSize otherwise)."""
        if not isinstance(shard_len, int):
            lengths = {int(n) for n in shard_len}
            if len(lengths) != 1:
                raise SwecError(-6, "shards are of different sizes (ErrShardSize)")
            shard_len = lengths.pop()
        if len(sketches) != self.total_shards:
            raise SwecError(-1, f"need {self.total_shards} sketches, got {len(sketches)}")
        n_pages = (shard_len + 4095) // 4096
        keep = []
        for s in sketches:
            if s is not None:
                s = np.ascontiguousarray(s, dtype=np.uint64)
                if s.shape != (n_pages,):
                    raise SwecError(-1, f"a sketch array must hold {n_pages} words, got {s.shape}")
            keep.append(s)
        return shard_len, n_pages, _ptrs(keep), keep

    def synchronize(self, stream: int = 0) -> None:
        check(lib().swec_stream_synchronize(self._h, stream))

    # Go spellings
    Encode, Reconstruct, ReconstructData, Verify = encode, reconstruct, reconstruct_data, verify


class EncoderGroup:
    """Several Encoder handles (one per GPU) behind the Encoder interface: every host-buffer call is split
    by byte-column range across the handles (swec_encode_multi / swec_reconstruct_multi)."""

    def __init__(self, data_shards: int, parity_shards: int, devices: list[int]):
        self.encoders = [Encoder(data_shards, parity_shards, d) for d in devices]
        self.data_shards, self.parity_shards = data_shards, parity_shards
        self._arr = (C.c_void_p * len(self.encoders))(*[e._h for e in self.encoders])

    @property
    def total_shards(self) -> int:
        return self.data_shards + self.parity_shards

    def close(self) -> None:
        for e in self.encoders:
            e.close()
        self.encoders = []

    def encode(self, shards: list[np.ndarray]) -> None:
        n = self.encoders[0]._check_shards(shards, allow_missing=False)
        check(lib().swec_encode_multi(self._arr, len(self.encoders), _ptrs(shards), n))

    def reconstruct(self, shards: list, data_only: bool = False) -> None:
        e0 = self.encoders[0]
        n = e0._check_shards(shards, allow_missing=True)
        present, ptrs = _fill_missing(shards, n, self.data_shards, data_only)
        check(lib().swec_reconstruct_multi(self._arr, len(self.encoders), ptrs, present.ctypes.data, n, int(data_only)))

    Encode, Reconstruct = encode, reconstruct


@dataclass
class ECContext:
    """ec_context.go:11-46"""
    DataShards: int = DataShardsCount
    ParityShards: int = ParityShardsCount
    Collection: str = ""
    VolumeId: int = 0
    device: int = 0

    def Total(self) -> int:
        return self.DataShards + self.ParityShards

    def CreateEncoder(self) -> Encoder:
        return Encoder(self.DataShards, self.ParityShards, self.device)

    def ToExt(self, shard_index: int) -> str:
        return ".ec%02d" % shard_index

    def String(self) -> str:
        return "%d+%d (total: %d)" % (self.DataShards, self.ParityShards, self.Total())


def NewDefaultECContext(collection: str = "", volume_id: int = 0, device: int = 0) -> ECContext:
    return ECContext(DataShardsCount, ParityShardsCount, collection, volume_id, device)


def ToExt(ec_index: int) -> str:
    return ".ec%02d" % ec_index


# ---- file level ---------------------------------------------------------------------------------

def generate_ec_files(base_file_name: str, buffer_size: int, large_block_size: int, small_block_size: int,
                      ctx: ECContext | None = None) -> None:
    ctx = ctx or NewDefaultECContext()
    check(lib().swec_generate_ec_files(base_file_name.encode(), buffer_size, large_block_size, small_block_size,
                                       ctx.DataShards, ctx.ParityShards, ctx.device))


def write_ec_files(base_file_name: str, ctx: ECContext | None = None) -> None:
    generate_ec_files(base_file_name, 256 * 1024, ErasureCodingLargeBlockSize, ErasureCodingSmallBlockSize, ctx)


def rebuild_ec_files(base_file_name: str, additional_dirs: list[str] | None = None,
                     ctx: ECContext | None = None, device: int = 0) -> list[int]:
    """RebuildEcFiles (ctx None ⇒ ratio from .vif or 10+4) / RebuildEcFilesWithContext."""
    arr, nd = _dirs(additional_dirs)
    ids = (C.c_uint32 * MaxShardCount)()
    n = C.c_int(0)
    check(lib().swec_rebuild_ec_files(base_file_name.encode(), arr, nd, *_code(ctx, device), ids, C.byref(n)))
    return list(ids[: n.value])


def verify_ec_files(base_file_name: str, additional_dirs: list[str] | None = None, ctx: ECContext | None = None,
                    device: int = 0):
    """Parity scrub of a shard set: returns (ok, mismatching 16-byte vectors per parity shard)."""
    arr, nd = _dirs(additional_dirs)
    bad = (C.c_uint64 * MaxShardCount)()
    ok = C.c_int(0)
    check(lib().swec_verify_ec_files(base_file_name.encode(), arr, nd, *_code(ctx, device), bad, C.byref(ok)))
    nm = ctx.ParityShards if ctx else ParityShardsCount
    return bool(ok.value), list(bad[:nm])


def page_sketch_file(path: str, seed: int, device: int = 0) -> tuple[np.ndarray, int]:
    """The page sketches of one shard file (swec_page_sketch_file): (uint64 array of ceil(len / 4096) words, len).  The
    file is only read; "file_direct_io" bit 0 reads it with O_DIRECT."""
    import os
    cap = (os.stat(path).st_size + 4095) // 4096
    while True:
        out = np.zeros(max(1, cap), dtype=np.uint64)
        shard_len, n = C.c_int64(0), C.c_int64(0)
        check(lib().swec_page_sketch_file(path.encode(), device, seed, out.ctypes.data, cap, C.byref(shard_len),
                                          C.byref(n)))
        if n.value <= cap:   # else the file grew since the stat: again with room for every page
            return out[:n.value], int(shard_len.value)
        cap = n.value


def _sketch_pages(pages):
    """The ctypes array of a "pages" list [(page, blamed mask, uncorrectable)] of the sketch locate calls, and its length."""
    pages = list(pages)
    arr = (SketchPage * max(1, len(pages)))()
    for a, (g, mask, unc) in zip(arr, pages):
        a.page, a.blamed_mask, a.uncorrectable = g, mask, int(unc)
    return arr, len(pages)


def sketch_needle_damage(pages, shard_len: int, dat_size: int, records, data_shards: int = DataShardsCount,
                         parity_shards: int = ParityShardsCount, large_block: int = ErasureCodingLargeBlockSize,
                         small_block: int = ErasureCodingSmallBlockSize, device: int = 0) -> dict:
    """Which records the pages flagged by Encoder.locate_sketch_damage[_checked] hit (swec_sketch_needle_damage), for
    shards of the volume image of dat_size bytes striped with large_block / small_block (shard_len must be its shard
    size).  records: (needle_id, offset, size) of every live record, sized as needle version 3.  Returns "needles" (one
    dict per record, in order, zero counts included) and "unowned" = [damaged, uncorrectable].  The counts are
    page-granular upper bounds (include/swec.h)."""
    arr, n_pages = _sketch_pages(pages)
    records = list(records)
    recs = (NeedleDamage * max(1, len(records)))()
    for r, (nid, off, size) in zip(recs, records):
        r.needle_id, r.offset, r.size = nid, off, size
    unowned = (C.c_uint64 * 2)()
    check(lib().swec_sketch_needle_damage(device, data_shards, parity_shards, shard_len, dat_size, large_block,
                                          small_block, arr, n_pages, recs, len(records), unowned))
    return {"needles": _needle_damage(recs[:len(records)]), "unowned": [int(unowned[0]), int(unowned[1])]}


def _sketch_result(ok, n, pages, per_shard) -> dict:
    return {"ok": bool(ok.value), "n_flagged": int(n.value),
            "pages": [(int(p.page), int(p.blamed_mask), bool(p.uncorrectable)) for p in pages[:n.value]],
            "shard_pages": {i: int(per_shard[i]) for i in range(MaxShardCount) if per_shard[i]}}


class _DamageOut:
    """The report out-parameters of a damage call: `args` are its four ctypes arguments (report, ranges, ranges_cap,
    n_ranges), result() the report, the first max_ranges ranges and their total as a dict."""

    def __init__(self, max_ranges: int):
        self.report, self.ranges, self.n = DamageReport(), (DamageRange * max(1, max_ranges))(), C.c_int(0)
        self.max_ranges = max_ranges
        self.args = (C.byref(self.report), self.ranges, max_ranges, C.byref(self.n))

    def result(self) -> dict:
        report, n_ranges = self.report, self.n.value
        shards = {i: (int(report.shard_bytes[i]), int(report.shard_first[i]), int(report.shard_last[i]))
                  for i in range(MaxShardCount) if report.shard_bytes[i]}
        return {"columns": int(report.columns), "damaged_columns": int(report.damaged_columns),
                "uncorrectable_columns": int(report.uncorrectable_columns),
                "first_uncorrectable": int(report.first_uncorrectable),
                "last_uncorrectable": int(report.last_uncorrectable), "shards": shards,
                "ranges": [(r.shard_id, r.offset, r.length) for r in self.ranges[:min(n_ranges, self.max_ranges)]],
                "n_ranges": n_ranges}


def _needle_damage(recs) -> list[dict]:
    return [{"needle_id": int(r.needle_id), "offset": int(r.offset), "size": int(r.size), "shard_mask": int(r.shard_mask),
             "damaged_bytes": int(r.damaged_bytes), "uncorrectable_bytes": int(r.uncorrectable_bytes)} for r in recs]


def locate_ec_damage(base_file_name: str, additional_dirs: list[str] | None = None, ctx: ECContext | None = None,
                     device: int = 0, radius: int = 1, max_ranges: int = 4096) -> dict:
    """Which shard files are wrong where parity does not match (swec_locate_ec_damage).  Returns ok, the column
    counts, "shards" = {shard id: (bytes blamed, first offset, last offset)} for the shards with damage, the
    uncorrectable summary, "ranges" = [(shard id or -1, offset, length)] (the first max_ranges) and "n_ranges"."""
    arr, nd = _dirs(additional_dirs)
    out, ok = _DamageOut(max_ranges), C.c_int(0)
    check(lib().swec_locate_ec_damage(base_file_name.encode(), arr, nd, *_code(ctx, device), radius, *out.args, C.byref(ok)))
    return {"ok": bool(ok.value), **out.result()}


def repair_ec_damage(base_file_name: str, additional_dirs: list[str] | None = None, ctx: ECContext | None = None,
                     device: int = 0, radius: int = 1, max_ranges: int = 4096) -> dict:
    """locate_ec_damage, which also corrects the located bytes in the shard files (swec_repair_ec_damage): only the
    blamed shards' damaged pages are rewritten.  Returns the report of the files as they were; "ok" is True iff no
    uncorrectable column remains.  Radius 2 can miscorrect a column with 3 or more wrong shards (include/swec.h)."""
    arr, nd = _dirs(additional_dirs)
    out, ok = _DamageOut(max_ranges), C.c_int(0)
    check(lib().swec_repair_ec_damage(base_file_name.encode(), arr, nd, *_code(ctx, device), radius, *out.args, C.byref(ok)))
    return {"ok": bool(ok.value), **out.result()}


def rebuild_ec_files_checked(base_file_name: str, additional_dirs: list[str] | None = None,
                             ctx: ECContext | None = None, device: int = 0, radius: int = 1,
                             max_ranges: int = 4096) -> dict:
    """rebuild_ec_files that reads every present shard and corrects the damage it locates in the shards it rebuilds
    from (swec_rebuild_ec_files_checked).  Returns "rebuilt" (the ids), "ok" (True iff something could be checked and
    no column is uncorrectable) and the report of locate_ec_damage over the present shards.  Radius 0 only detects;
    run repair_ec_damage afterwards to fix the present shards (include/swec.h)."""
    arr, nd = _dirs(additional_dirs)
    ids, n_ids = (C.c_uint32 * MaxShardCount)(), C.c_int(0)
    out, ok = _DamageOut(max_ranges), C.c_int(0)
    check(lib().swec_rebuild_ec_files_checked(base_file_name.encode(), arr, nd, *_code(ctx, device), radius, ids,
                                              C.byref(n_ids), *out.args, C.byref(ok)))
    return {"rebuilt": list(ids[: n_ids.value]), "ok": bool(ok.value), **out.result()}


def heal_ec_files(base_file_name: str, additional_dirs: list[str] | None = None, ctx: ECContext | None = None,
                  device: int = 0, radius: int = 1, max_ranges: int = 4096) -> dict:
    """rebuild_ec_files_checked that also corrects the damage it locates in the present shard files, in one full read
    (swec_heal_ec_files): only the blamed shards' flagged pages are rewritten, and uncorrectable columns are left as
    found.  Returns what rebuild_ec_files_checked returns for the same files (include/swec.h)."""
    arr, nd = _dirs(additional_dirs)
    ids, n_ids = (C.c_uint32 * MaxShardCount)(), C.c_int(0)
    out, ok = _DamageOut(max_ranges), C.c_int(0)
    check(lib().swec_heal_ec_files(base_file_name.encode(), arr, nd, *_code(ctx, device), radius, ids, C.byref(n_ids),
                                   *out.args, C.byref(ok)))
    return {"rebuilt": list(ids[: n_ids.value]), "ok": bool(ok.value), **out.result()}


def _check_decoded(status: int, out: _DamageOut) -> None:
    """check(), but a SWEC_ERR_UNCORRECTABLE error carries the report as .report"""
    if STATUS.get(status) == "SWEC_ERR_UNCORRECTABLE":
        err = SwecError(status, lib().swec_last_error().decode(errors="replace"))
        err.report = out.result()
        raise err
    check(status)


def write_dat_file_checked(base_file_name: str, dat_file_size: int, shard_file_names: list, data_shards: int = DataShardsCount,
                           parity_shards: int = ParityShardsCount, large_block: int = ErasureCodingLargeBlockSize,
                           small_block: int = ErasureCodingSmallBlockSize, device: int = 0, radius: int = 1,
                           max_ranges: int = 4096) -> dict:
    """write_dat_file from any k of the k+m shards (swec_write_dat_file_checked): shard_file_names has k+m entries, None
    for a missing shard.  Damaged data shards are corrected, and missing ones rebuilt, on the GPU before the .dat is
    written.  Returns "dat_file_size", "ok" (True iff something could be checked and nothing is uncorrectable) and the
    report of rebuild_ec_files_checked.  Uncorrectable columns raise SwecError(SWEC_ERR_UNCORRECTABLE), with the report
    in its .report, and leave no .dat (include/swec.h)."""
    names = (C.c_char_p * len(shard_file_names))(*[s.encode() if s else None for s in shard_file_names])
    out, ok = _DamageOut(max_ranges), C.c_int(0)
    _check_decoded(lib().swec_write_dat_file_checked(base_file_name.encode(), dat_file_size, names, data_shards, parity_shards,
                                                     large_block, small_block, device, radius, *out.args, C.byref(ok)), out)
    return {"dat_file_size": dat_file_size, "ok": bool(ok.value), **out.result()}


def write_dat_file(base_file_name: str, dat_file_size: int, shard_file_names: list[str],
                   data_shards: int = DataShardsCount, large_block: int = ErasureCodingLargeBlockSize,
                   small_block: int = ErasureCodingSmallBlockSize) -> None:
    names = (C.c_char_p * len(shard_file_names))(*[s.encode() for s in shard_file_names])
    check(lib().swec_write_dat_file(base_file_name.encode(), dat_file_size, names, data_shards, large_block, small_block))


# ---- whole-volume operations (the file work of the three EC gRPC handlers) --------------------------

def _dirs(additional_dirs):
    dirs = [d.encode() for d in (additional_dirs or [])]
    return ((C.c_char_p * max(1, len(dirs)))(*dirs) if dirs else None), len(dirs)


def _code(ctx: ECContext | None, device: int):
    """(k, m, device) of a file call: the context's, or 0, 0 (the ratio from .vif, else 10+4) and `device`."""
    return (ctx.DataShards, ctx.ParityShards, ctx.device) if ctx else (0, 0, device)


def volume_ec_shards_generate(data_base_file_name: str, index_base_file_name: str | None = None,
                              needle_version: int = 0, expire_at_sec: int = 0, device: int = 0) -> None:
    """VolumeEcShardsGenerate (volume_grpc_erasure_coding.go:43-146): .ecx first, shards, .vif; cleanup on error."""
    check(lib().swec_ec_shards_generate(data_base_file_name.encode(),
                                        (index_base_file_name or "").encode(), needle_version, expire_at_sec, device))


def volume_ec_shards_rebuild(data_base_file_name: str, index_base_file_name: str | None = None,
                             additional_dirs: list[str] | None = None, device: int = 0) -> list[int]:
    """VolumeEcShardsRebuild (volume_grpc_erasure_coding.go:149-225): RebuildEcFiles + RebuildEcxFile."""
    arr, n = _dirs(additional_dirs)
    ids = (C.c_uint32 * MaxShardCount)()
    cnt = C.c_int(0)
    check(lib().swec_ec_shards_rebuild(data_base_file_name.encode(), (index_base_file_name or "").encode(),
                                       arr, n, device, ids, C.byref(cnt)))
    return list(ids[: cnt.value])


def volume_ec_shards_heal(data_base_file_name: str, index_base_file_name: str | None = None,
                          additional_dirs: list[str] | None = None, device: int = 0, radius: int = 1,
                          max_ranges: int = 4096) -> dict:
    """volume_ec_shards_rebuild through heal_ec_files (swec_ec_shards_heal): the lost shards rebuilt and the damaged
    present ones corrected, then RebuildEcxFile.  Returns what heal_ec_files returns."""
    arr, nd = _dirs(additional_dirs)
    ids, n_ids = (C.c_uint32 * MaxShardCount)(), C.c_int(0)
    out, ok = _DamageOut(max_ranges), C.c_int(0)
    check(lib().swec_ec_shards_heal(data_base_file_name.encode(), (index_base_file_name or "").encode(), arr, nd, device,
                                    radius, ids, C.byref(n_ids), *out.args, C.byref(ok)))
    return {"rebuilt": list(ids[: n_ids.value]), "ok": bool(ok.value), **out.result()}


def volume_ec_shards_to_volume(data_base_file_name: str, index_base_file_name: str | None = None,
                               additional_dirs: list[str] | None = None) -> int:
    """VolumeEcShardsToVolume (volume_grpc_erasure_coding.go:578-668): shards + .ecx/.ecj → .dat + .idx.
    Returns the .dat size; raises SwecError(SWEC_ERR_NO_LIVE_NEEDLES) for an all-deleted volume."""
    arr, n = _dirs(additional_dirs)
    size = C.c_int64(0)
    check(lib().swec_ec_shards_to_volume(data_base_file_name.encode(), (index_base_file_name or "").encode(),
                                         arr, n, C.byref(size)))
    return int(size.value)


def ec_shards_to_volume_checked(data_base_file_name: str, index_base_file_name: str | None = None,
                                additional_dirs: list[str] | None = None, device: int = 0, radius: int = 1,
                                max_ranges: int = 4096) -> dict:
    """volume_ec_shards_to_volume from any k of the k+m shards, correcting damaged data shards on the GPU before the
    .dat is written (swec_ec_shards_to_volume_checked).  Returns "dat_file_size", "ok" and the report, as
    write_dat_file_checked does; uncorrectable columns raise SwecError(SWEC_ERR_UNCORRECTABLE) with .report and leave
    neither .dat nor .idx, so the EC shards should be kept."""
    arr, nd = _dirs(additional_dirs)
    size, out, ok = C.c_int64(0), _DamageOut(max_ranges), C.c_int(0)
    _check_decoded(lib().swec_ec_shards_to_volume_checked(data_base_file_name.encode(), (index_base_file_name or "").encode(),
                                                          arr, nd, device, radius, C.byref(size), *out.args, C.byref(ok)),
                   out)
    return {"dat_file_size": int(size.value), "ok": bool(ok.value), **out.result()}


def _needle_reads(needle_ids, capacity, sizes=None):
    """capacity: fixed bytes per needle, or None with `sizes` (exact bytes per needle from a sizing pass)."""
    reads = (NeedleRead * len(needle_ids))()
    caps = [capacity] * len(needle_ids) if sizes is None else list(sizes)
    starts = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
    arena = np.empty(max(1, int(starts[-1])), dtype=np.uint8)
    for j, (r, nid) in enumerate(zip(reads, needle_ids)):
        r.needle_id, r.buf, r.capacity = nid, arena.ctypes.data + int(starts[j]), caps[j]
    return reads, arena, starts


def _needle_results(reads, arena, starts):
    return [{"id": r.needle_id, "status": STATUS.get(r.status, str(r.status)), "offset": r.offset, "size": r.size,
             "bytes": arena[int(starts[j]): int(starts[j]) + r.n_bytes] if r.status == 0 else None,
             "n_bytes": r.n_bytes, "recovered_intervals": r.n_recovered_intervals} for j, r in enumerate(reads)]


def _read_needles(call, needle_ids, capacity):
    """capacity None ⇒ two passes: a sizing pass with zero-capacity buffers (every live needle answers
    SWEC_ERR_INVALID_ARG with the bytes it needs, nothing is read), then the real one into an exact arena."""
    if capacity is None:
        reads, arena, starts = _needle_reads(needle_ids, 0)
        check(call(reads, len(needle_ids)))
        sizes = [r.n_bytes if r.status == -1 else 0 for r in reads]
        reads, arena, starts = _needle_reads(needle_ids, None, sizes)
    else:
        reads, arena, starts = _needle_reads(needle_ids, capacity)
    check(call(reads, len(needle_ids)))
    return _needle_results(reads, arena, starts)


class EcVolume:
    """A mounted EC volume (erasure_coding.EcVolume, ec_volume.go:36-160) for the read path: shard files open,
    .ecx loaded, the encoder behind degraded reads kept warm.  ReadEcShardNeedles = Store.ReadEcShardNeedle
    (store_ec.go:252-355) for many needles in one call."""

    def __init__(self, data_base_file_name: str, index_base_file_name: str | None = None,
                 additional_dirs: list[str] | None = None, device: int = 0):
        arr, n = _dirs(additional_dirs)
        h = C.c_void_p()
        check(lib().swec_ec_volume_open(data_base_file_name.encode(), (index_base_file_name or "").encode(), arr, n,
                                        device, C.byref(h)))
        self._h = h

    def read_needles(self, needle_ids: list[int], capacity: int | None = None):
        return _read_needles(lambda reads, n: lib().swec_ec_volume_read_needles(self._h, reads, n), needle_ids, capacity)

    def delete_needle(self, needle_id: int) -> None:
        """DeleteNeedleFromEcx (ec_volume_delete.go:28-93)"""
        check(lib().swec_ec_volume_delete_needle(self._h, needle_id))

    DeleteNeedleFromEcx = delete_needle

    def info(self) -> dict:
        k, m, ver, bits, sds = C.c_int(0), C.c_int(0), C.c_int(0), C.c_uint32(0), C.c_int64(0)
        check(lib().swec_ec_volume_info(self._h, C.byref(k), C.byref(m), C.byref(ver), C.byref(sds), C.byref(bits)))
        return {"data_shards": k.value, "parity_shards": m.value, "version": ver.value, "shard_dat_size": sds.value,
                "local_shards": [i for i in range(32) if bits.value >> i & 1]}

    def file_and_delete_count(self) -> tuple[int, int]:
        """FileAndDeleteCount (ec_volume.go:330-349)"""
        f, d = C.c_uint64(0), C.c_uint64(0)
        check(lib().swec_ec_volume_counts(self._h, C.byref(f), C.byref(d)))
        return int(f.value), int(d.value)

    FileAndDeleteCount = file_and_delete_count

    def scrub_local(self):
        """ScrubLocal (ec_volume_scrub.go:27-118): (entries walked, broken shard ids, findings)."""
        n, nb, ne = C.c_int64(0), C.c_int(0), C.c_int(0)
        broken = (C.c_uint32 * MaxShardCount)()
        buf = C.create_string_buffer(1 << 20)
        check(lib().swec_ec_volume_scrub_local(self._h, C.byref(n), broken, C.byref(nb), buf, len(buf), C.byref(ne)))
        return int(n.value), list(broken[: nb.value]), (buf.value.decode().split("\n") if ne.value else [])

    ScrubLocal = scrub_local

    def scrub_needles(self, volume_id: int = 0):
        """The whole ScrubLocal: scrub_local's walk plus Needle.ReadBytes (size, layout, CRC32-C) of every record whose
        chunks are all local, on the GPU.  Same result shape as scrub_local."""
        n, nb, ne = C.c_int64(0), C.c_int(0), C.c_int(0)
        broken = (C.c_uint32 * MaxShardCount)()
        buf = C.create_string_buffer(1 << 22)
        check(lib().swec_ec_volume_scrub_needles(self._h, volume_id, C.byref(n), broken, C.byref(nb), buf, len(buf),
                                                 C.byref(ne)))
        return int(n.value), list(broken[: nb.value]), (buf.value.decode().split("\n") if ne.value else [])

    def locate_needle_damage(self, radius: int = 1, max_ranges: int = 4096, max_needles: int = 1 << 16) -> dict:
        """locate_ec_damage on the volume's shards (all k+m must be local), and which live needles the damage hits
        (swec_ec_volume_locate_needle_damage).  Returns the locate_ec_damage dict plus "needles" (ascending id, the first
        max_needles of those with a non-zero count: needle_id, offset, size, shard_mask, damaged_bytes — a repair
        restores them — and uncorrectable_bytes — it cannot), "n_needles" and "unowned" = [damaged, uncorrectable] bytes
        that no live needle owns.  The shard files are only read."""
        out, ok = _DamageOut(max_ranges), C.c_int(0)
        needles, n_needles, unowned = (NeedleDamage * max(1, max_needles))(), C.c_int(0), (C.c_uint64 * 2)()
        check(lib().swec_ec_volume_locate_needle_damage(self._h, radius, *out.args, needles, max_needles,
                                                        C.byref(n_needles), unowned, C.byref(ok)))
        return {"ok": bool(ok.value), **out.result(),
                "needles": _needle_damage(needles[:min(n_needles.value, max_needles)]), "n_needles": n_needles.value,
                "unowned": [int(unowned[0]), int(unowned[1])]}

    LocateNeedleDamage = locate_needle_damage

    def repair_needle_damage(self, radius: int = 1, max_ranges: int = 4096, max_needles: int = 1 << 16) -> dict:
        """locate_needle_damage and repair_ec_damage in one pass over the volume's shards, written to the files the
        handle reads, then every named needle checked again from the repaired files like scrub_needles checks it
        (swec_ec_volume_repair_needle_damage).  Returns the locate_needle_damage dict, as it was before the call; each
        needle also carries its check: status (0 ok, 1 size mismatch, 2 out of range, 3 bad crc, 4 outside image),
        range_index, data_size, crc_got, crc_want and legacy_crc.  "ok" is True iff no uncorrectable column remains and
        every named needle (not only the first max_needles) checks ok: a column miscorrected beyond the guarantee of
        the code shows as a needle that does not."""
        from ._native import NeedleCheck
        out, ok = _DamageOut(max_ranges), C.c_int(0)
        needles, n_needles, unowned = (NeedleDamage * max(1, max_needles))(), C.c_int(0), (C.c_uint64 * 2)()
        checks = (NeedleCheck * max(1, max_needles))()
        check(lib().swec_ec_volume_repair_needle_damage(self._h, radius, *out.args, needles, checks, max_needles,
                                                        C.byref(n_needles), unowned, C.byref(ok)))
        shown = min(n_needles.value, max_needles)
        named = [{**d, "status": int(c.status), "range_index": int(c.range_index), "data_size": int(c.data_size),
                  "crc_got": int(c.crc_got), "crc_want": int(c.crc_want), "legacy_crc": int(c.legacy_crc)}
                 for d, c in zip(_needle_damage(needles[:shown]), checks[:shown])]
        return {"ok": bool(ok.value), **out.result(), "needles": named,
                "n_needles": n_needles.value, "unowned": [int(unowned[0]), int(unowned[1])]}

    RepairNeedleDamage = repair_needle_damage

    def page_sketch(self, seed: int, shards=None) -> tuple[dict, int]:
        """The page sketches of local shards, read through the handle under its lock so that they never overlap a
        repair through it (swec_ec_volume_page_sketch): ({shard id: uint64 array of ceil(len / 4096) words}, len).
        shards: the shard ids to sketch (None: every local shard), all in one file pipeline pass."""
        info = self.info()
        ids = info["local_shards"] if shards is None else list(shards)
        total = info["data_shards"] + info["parity_shards"]
        cap = (info["shard_dat_size"] + ErasureCodingSmallBlockSize + 4096) // 4096   # the shards' pages, or more
        while True:
            out = {i: np.zeros(max(1, cap), dtype=np.uint64) for i in ids}
            ptrs = (C.c_void_p * total)(*[out[i].ctypes.data if i in out else None for i in range(total)])
            shard_len, n = C.c_int64(0), C.c_int64(0)
            check(lib().swec_ec_volume_page_sketch(self._h, seed, ptrs, cap, C.byref(shard_len), C.byref(n)))
            if n.value <= cap:
                return {i: a[:n.value] for i, a in out.items()}, int(shard_len.value)
            cap = n.value

    def sketch_needle_damage(self, pages, shard_len: int, max_needles: int = 1 << 16) -> dict:
        """Which live needles the pages flagged by Encoder.locate_sketch_damage[_checked] (their "pages" list, for
        shards of shard_len bytes) hit, from the .ecx alone (swec_ec_volume_sketch_needle_damage): no local shard is
        needed.  Returns "needles" (ascending id, the first max_needles of those with a non-zero count), "n_needles" and
        "unowned" = [damaged, uncorrectable].  The counts are page-granular upper bounds (include/swec.h)."""
        arr, n_pages = _sketch_pages(pages)
        needles, n_needles, unowned = (NeedleDamage * max(1, max_needles))(), C.c_int(0), (C.c_uint64 * 2)()
        check(lib().swec_ec_volume_sketch_needle_damage(self._h, shard_len, arr, n_pages, needles, max_needles,
                                                        C.byref(n_needles), unowned))
        return {"needles": _needle_damage(needles[:min(n_needles.value, max_needles)]), "n_needles": n_needles.value,
                "unowned": [int(unowned[0]), int(unowned[1])]}

    PageSketch, SketchNeedleDamage = page_sketch, sketch_needle_damage

    def close(self) -> None:
        h, self._h = getattr(self, "_h", None), None
        if h and callable(lib):
            lib().swec_ec_volume_close(h)

    __del__ = close
    ReadEcShardNeedles = read_needles


def check_needles_device(dat_ptr: int, dat_size: int, records, needle_version: int = 3, device: int = 0,
                         stream: int | None = None) -> list[dict]:
    """Needle.ReadBytes on records of a volume image in device memory (swec_check_needles_device).  records: iterable
    of (needle_id, offset, size).  One dict per record: status (0 ok, 1 size mismatch, 2 out of range, 3 bad crc,
    4 outside image), range_index, data_size, crc_got, crc_want, legacy_crc."""
    from ._native import NeedleCheck
    records = list(records)
    arr = (NeedleCheck * max(1, len(records)))()
    for c, (nid, off, size) in zip(arr, records):
        c.needle_id, c.offset, c.size = nid, off, size
    check(lib().swec_check_needles_device(device, dat_ptr, dat_size, needle_version, arr, len(records), stream))
    return [{"needle_id": c.needle_id, "status": c.status, "range_index": c.range_index, "data_size": c.data_size,
             "crc_got": c.crc_got, "crc_want": c.crc_want, "legacy_crc": c.legacy_crc} for c in arr[:len(records)]]


def read_ec_shard_needles(data_base_file_name: str, needle_ids: list[int], index_base_file_name: str | None = None,
                          additional_dirs: list[str] | None = None, device: int = 0, capacity: int | None = None):
    """One-shot form: mount, read, unmount.  Returns one dict per id with status name, offset, size, the raw
    record bytes and how many intervals had to be reconstructed."""
    arr, n = _dirs(additional_dirs)
    return _read_needles(lambda reads, cnt: lib().swec_read_ec_needles(
        data_base_file_name.encode(), (index_base_file_name or "").encode(), arr, n, reads, cnt, device),
        needle_ids, capacity)


ReadEcShardNeedles = read_ec_shard_needles
VolumeEcShardsGenerate, VolumeEcShardsRebuild, VolumeEcShardsToVolume = (
    volume_ec_shards_generate, volume_ec_shards_rebuild, volume_ec_shards_to_volume)


# ---- index files (.idx / .ecx / .ecj) --------------------------------------------------------------

def write_sorted_file_from_idx(base_file_name: str, ext: str = ".ecx") -> None:
    """WriteSortedFileFromIdx (ec_encoder.go:31-58)"""
    check(lib().swec_write_sorted_file_from_idx(base_file_name.encode(), ext.encode()))


def rebuild_ecx_file(base_file_name: str) -> None:
    """RebuildEcxFile (ec_volume_delete.go:95-142)"""
    check(lib().swec_rebuild_ecx_file(base_file_name.encode()))


def write_idx_file_from_ec_index(base_file_name: str) -> None:
    """WriteIdxFileFromEcIndex (ec_decoder.go:35-60)"""
    check(lib().swec_write_idx_file_from_ec_index(base_file_name.encode()))


def check_index_file(path: str, needle_version: int = 3) -> tuple[int, list[str]]:
    """idx.CheckIndexFile (weed/storage/idx/check.go:36-111): (entries processed, findings)."""
    n, k = C.c_int64(0), C.c_int(0)
    buf = C.create_string_buffer(1 << 20)
    check(lib().swec_check_index_file(path.encode(), needle_version, C.byref(n), buf, len(buf), C.byref(k)))
    text = buf.value.decode()
    return int(n.value), (text.split("\n") if k.value else [])


CheckIndexFile = check_index_file


def has_live_needles(index_base_file_name: str) -> bool:
    v = C.c_int(0)
    check(lib().swec_has_live_needles(index_base_file_name.encode(), C.byref(v)))
    return bool(v.value)


def find_dat_file_size(data_base_file_name: str, index_base_file_name: str) -> int:
    v = C.c_int64(0)
    check(lib().swec_find_dat_file_size(data_base_file_name.encode(), index_base_file_name.encode(), C.byref(v)))
    return int(v.value)


WriteSortedFileFromIdx, RebuildEcxFile, WriteIdxFileFromEcIndex = (write_sorted_file_from_idx, rebuild_ecx_file,
                                                                    write_idx_file_from_ec_index)
HasLiveNeedles, FindDatFileSize = has_live_needles, find_dat_file_size
WriteEcFiles, WriteEcFilesWithContext = write_ec_files, write_ec_files
generateEcFiles, RebuildEcFiles, WriteDatFile = generate_ec_files, rebuild_ec_files, write_dat_file


# ---- layout --------------------------------------------------------------------------------------

def expected_shard_size(dat_size: int, data_shards: int = DataShardsCount,
                        large_block: int = ErasureCodingLargeBlockSize,
                        small_block: int = ErasureCodingSmallBlockSize) -> int:
    return int(lib().swec_expected_shard_size(dat_size, data_shards, large_block, small_block))


def locate_data(large_block_length: int, small_block_length: int, shard_dat_size: int, offset: int, size: int,
                data_shards: int = DataShardsCount):
    """LocateData → list of (BlockIndex, InnerBlockOffset, Size, IsLargeBlock, LargeBlockRowsCount)."""
    cap = 4 + int(size // max(1, small_block_length)) + 2
    buf = (Interval * cap)()
    n = lib().swec_locate_data(large_block_length, small_block_length, shard_dat_size, offset, size,
                               data_shards, buf, cap)
    if n < 0:
        check(n)
    return [(b.block_index, b.inner_block_offset, b.size, bool(b.is_large_block), b.large_block_rows_count)
            for b in buf[:n]]


def interval_to_shard(iv, large_block: int, small_block: int, data_shards: int = DataShardsCount):
    """Interval.ToShardIdAndOffset"""
    c = Interval(iv[0], int(iv[3]), iv[1], iv[2], iv[4], 0)
    sid, off = C.c_int(0), C.c_int64(0)
    lib().swec_interval_to_shard(C.byref(c), large_block, small_block, data_shards, C.byref(sid), C.byref(off))
    return sid.value, off.value


LocateData = locate_data
