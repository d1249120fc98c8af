"""ctypes binding of libswec.so — one prototype per function declared in include/swec.h."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(HERE, "libswec.so")
_lib = None

SWEC_MAX_SHARDS = 32

STATUS = {
    0: "SWEC_OK", -1: "SWEC_ERR_INVALID_ARG", -2: "SWEC_ERR_TOO_FEW_SHARDS", -3: "SWEC_ERR_CUDA",
    -4: "SWEC_ERR_IO", -5: "SWEC_ERR_NOMEM", -6: "SWEC_ERR_SHARD_SIZE", -7: "SWEC_ERR_NO_DEVICE",
    -8: "SWEC_ERR_JIT", -9: "SWEC_ERR_NO_LIVE_NEEDLES",
    -10: "SWEC_ERR_NOT_FOUND", -11: "SWEC_ERR_DELETED", -12: "SWEC_ERR_UNCORRECTABLE",
}


class SwecError(RuntimeError):
    def __init__(self, status: int, detail: str = ""):
        self.status = status
        self.name = STATUS.get(status, str(status))
        super().__init__(f"{self.name}: {detail}" if detail else self.name)


class ReconstructItem(C.Structure):
    _fields_ = [("shards", C.POINTER(C.c_void_p)), ("present", C.POINTER(C.c_uint8)),
                ("shard_len", C.c_size_t), ("data_only", C.c_int)]


class Interval(C.Structure):
    _fields_ = [("block_index", C.c_int32), ("is_large_block", C.c_int32),
                ("inner_block_offset", C.c_int64), ("size", C.c_int64),
                ("large_block_rows_count", C.c_int32), ("reserved", C.c_int32)]


class NeedleRead(C.Structure):
    _fields_ = [("needle_id", C.c_uint64), ("buf", C.c_void_p), ("capacity", C.c_size_t), ("offset", C.c_int64),
                ("size", C.c_int32), ("status", C.c_int32), ("n_bytes", C.c_size_t),
                ("n_recovered_intervals", C.c_int32), ("reserved", C.c_int32)]


class NeedleCheck(C.Structure):
    _fields_ = [("needle_id", C.c_uint64), ("offset", C.c_int64), ("size", C.c_int32), ("status", C.c_int32),
                ("range_index", C.c_int32), ("data_size", C.c_uint32), ("crc_got", C.c_uint32), ("crc_want", C.c_uint32),
                ("legacy_crc", C.c_int32), ("reserved", C.c_int32)]


class DamageReport(C.Structure):
    _fields_ = [("columns", C.c_uint64), ("damaged_columns", C.c_uint64), ("uncorrectable_columns", C.c_uint64),
                ("first_uncorrectable", C.c_int64), ("last_uncorrectable", C.c_int64),
                ("shard_bytes", C.c_uint64 * SWEC_MAX_SHARDS), ("shard_first", C.c_int64 * SWEC_MAX_SHARDS),
                ("shard_last", C.c_int64 * SWEC_MAX_SHARDS)]


class DamageRange(C.Structure):
    _fields_ = [("shard_id", C.c_int32), ("reserved", C.c_int32), ("offset", C.c_int64), ("length", C.c_int64)]


class NeedleDamage(C.Structure):
    _fields_ = [("needle_id", C.c_uint64), ("offset", C.c_int64), ("size", C.c_int32), ("shard_mask", C.c_uint32),
                ("damaged_bytes", C.c_uint64), ("uncorrectable_bytes", C.c_uint64)]


class SketchPage(C.Structure):
    _fields_ = [("page", C.c_int64), ("blamed_mask", C.c_uint32), ("uncorrectable", C.c_int32)]


NEEDLE_STATUS = {0: "ok", 1: "size mismatch", 2: "out of range", 3: "bad crc", 4: "outside image"}


# name → (restype, argtypes); kept in step with include/swec.h (tests/test_abi.py checks both ways)
PROTOTYPES = {
    "swec_version": (C.c_char_p, []),
    "swec_strerror": (C.c_char_p, [C.c_int]),
    "swec_last_error": (C.c_char_p, []),
    "swec_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "swec_shutdown": (None, []),
    "swec_kernel_launches": (C.c_uint64, []),
    "swec_set_option": (C.c_int, [C.c_char_p, C.c_long]),
    "swec_device_spread_order": (C.c_int, [C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_int)]),
    "swec_debug_power_state": (C.c_int, [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int)]),
    "swec_jit_stats": (C.c_int, [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_int), C.POINTER(C.c_uint64)]),
    "swec_debug_jit_compile": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_size_t), C.POINTER(C.c_int),
                                         C.POINTER(C.c_int)]),
    "swec_encoder_new": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "swec_encoder_free": (None, [C.c_void_p]),
    "swec_encoder_matrix": (C.c_int, [C.c_void_p, C.c_void_p]),
    "swec_reconstruct_matrix": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                          C.POINTER(C.c_int), C.c_void_p]),
    "swec_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "swec_reconstruct": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    "swec_reconstruct_batch": (C.c_int, [C.c_void_p, C.POINTER(ReconstructItem), C.c_int]),
    "swec_encode_multi": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    "swec_reconstruct_multi": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]),
    "swec_alloc_pinned_shards": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]),
    "swec_verify": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_int)]),
    "swec_encode_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "swec_reconstruct_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "swec_apply_device": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "swec_encode_volume_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                            C.c_void_p, C.c_void_p]),
    "swec_extract_data_shard_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                                 C.c_int, C.c_void_p, C.c_void_p]),
    "swec_write_dat_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "swec_stream_synchronize": (C.c_int, [C.c_void_p, C.c_void_p]),
    "swec_write_ec_files": (C.c_int, [C.c_char_p, C.c_int]),
    "swec_generate_ec_files": (C.c_int, [C.c_char_p, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int]),
    "swec_rebuild_ec_files": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_void_p, C.POINTER(C.c_int)]),
    "swec_verify_ec_files": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                       C.POINTER(C.c_int)]),
    "swec_locate_ec_damage": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.POINTER(DamageReport), C.POINTER(DamageRange), C.c_int, C.POINTER(C.c_int),
                                        C.POINTER(C.c_int)]),
    "swec_locate_damage_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.POINTER(DamageReport),
                                            C.POINTER(DamageRange), C.c_int, C.POINTER(C.c_int), C.c_void_p]),
    "swec_repair_ec_damage": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.POINTER(DamageReport), C.POINTER(DamageRange), C.c_int, C.POINTER(C.c_int),
                                        C.POINTER(C.c_int)]),
    "swec_correct_damage_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.POINTER(DamageReport),
                                             C.POINTER(DamageRange), C.c_int, C.POINTER(C.c_int), C.c_void_p]),
    "swec_ec_volume_locate_needle_damage": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(DamageReport), C.POINTER(DamageRange),
                                                      C.c_int, C.POINTER(C.c_int), C.POINTER(NeedleDamage), C.c_int,
                                                      C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    "swec_ec_volume_repair_needle_damage": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(DamageReport), C.POINTER(DamageRange),
                                                      C.c_int, C.POINTER(C.c_int), C.POINTER(NeedleDamage),
                                                      C.POINTER(NeedleCheck), C.c_int, C.POINTER(C.c_int),
                                                      C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    "swec_locate_needle_damage_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int64, C.c_int64, C.c_int64,
                                                   C.c_int, C.POINTER(NeedleDamage), C.c_int, C.POINTER(DamageReport),
                                                   C.POINTER(DamageRange), C.c_int, C.POINTER(C.c_int),
                                                   C.POINTER(C.c_uint64), C.c_void_p]),
    "swec_rebuild_ec_files_checked": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                C.c_void_p, C.POINTER(C.c_int), C.POINTER(DamageReport),
                                                C.POINTER(DamageRange), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "swec_reconstruct_checked_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int,
                                                  C.POINTER(DamageReport), C.POINTER(DamageRange), C.c_int,
                                                  C.POINTER(C.c_int), C.c_void_p]),
    "swec_decode_data_checked_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int,
                                                  C.POINTER(DamageReport), C.POINTER(DamageRange), C.c_int,
                                                  C.POINTER(C.c_int), C.c_void_p]),
    "swec_heal_ec_files": (C.c_int, [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                     C.POINTER(C.c_int), C.POINTER(DamageReport), C.POINTER(DamageRange), C.c_int,
                                     C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "swec_heal_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.POINTER(DamageReport),
                                   C.POINTER(DamageRange), C.c_int, C.POINTER(C.c_int), C.c_void_p]),
    "swec_page_sketch_device": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_uint64, C.c_uint64, C.c_void_p,
                                          C.c_void_p]),
    "swec_page_sketch_file": (C.c_int, [C.c_char_p, C.c_int, C.c_uint64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64),
                                        C.POINTER(C.c_int64)]),
    "swec_locate_sketch_damage": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(SketchPage),
                                            C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    "swec_locate_sketch_damage_checked": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.POINTER(SketchPage),
                                                    C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_uint64), C.c_void_p,
                                                    C.POINTER(C.c_int)]),
    "swec_sketch_needle_damage": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
                                            C.POINTER(SketchPage), C.c_int64, C.POINTER(NeedleDamage), C.c_int,
                                            C.POINTER(C.c_uint64)]),
    "swec_ec_volume_page_sketch": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_int64, C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64)]),
    "swec_ec_volume_sketch_needle_damage": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(SketchPage), C.c_int64,
                                                      C.POINTER(NeedleDamage), C.c_int, C.POINTER(C.c_int),
                                                      C.POINTER(C.c_uint64)]),
    "swec_write_dat_file": (C.c_int, [C.c_char_p, C.c_int64, C.c_void_p, C.c_int, C.c_int64, C.c_int64]),
    "swec_write_dat_file_checked": (C.c_int, [C.c_char_p, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int64,
                                              C.c_int, C.c_int, C.POINTER(DamageReport), C.POINTER(DamageRange), C.c_int,
                                              C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "swec_ec_shards_generate": (C.c_int, [C.c_char_p, C.c_char_p, C.c_uint32, C.c_uint64, C.c_int]),
    "swec_ec_shards_rebuild": (C.c_int, [C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                         C.POINTER(C.c_int)]),
    "swec_ec_shards_heal": (C.c_int, [C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                      C.POINTER(C.c_int), C.POINTER(DamageReport), C.POINTER(DamageRange), C.c_int,
                                      C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "swec_ec_shards_to_volume": (C.c_int, [C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.POINTER(C.c_int64)]),
    "swec_ec_shards_to_volume_checked": (C.c_int, [C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                   C.POINTER(C.c_int64), C.POINTER(DamageReport), C.POINTER(DamageRange),
                                                   C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "swec_read_ec_needles": (C.c_int, [C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.POINTER(NeedleRead), C.c_int, C.c_int]),
    "swec_ec_volume_open": (C.c_int, [C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "swec_ec_volume_read_needles": (C.c_int, [C.c_void_p, C.POINTER(NeedleRead), C.c_int]),
    "swec_ec_volume_delete_needle": (C.c_int, [C.c_void_p, C.c_uint64]),
    "swec_ec_volume_scrub_local": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_uint32), C.POINTER(C.c_int),
                                             C.c_char_p, C.c_size_t, C.POINTER(C.c_int)]),
    "swec_ec_volume_scrub_needles": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(C.c_int64), C.POINTER(C.c_uint32),
                                               C.POINTER(C.c_int), C.c_char_p, C.c_size_t, C.POINTER(C.c_int)]),
    "swec_check_needles_device": (C.c_int, [C.c_int, C.c_void_p, C.c_int64, C.c_int, C.POINTER(NeedleCheck), C.c_int,
                                            C.c_void_p]),
    "swec_ec_volume_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                      C.POINTER(C.c_int64), C.POINTER(C.c_uint32)]),
    "swec_ec_volume_counts": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "swec_ec_volume_close": (None, [C.c_void_p]),
    "swec_write_sorted_file_from_idx": (C.c_int, [C.c_char_p, C.c_char_p]),
    "swec_rebuild_ecx_file": (C.c_int, [C.c_char_p]),
    "swec_write_idx_file_from_ec_index": (C.c_int, [C.c_char_p]),
    "swec_check_index_file": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(C.c_int64), C.c_char_p, C.c_size_t, C.POINTER(C.c_int)]),
    "swec_has_live_needles": (C.c_int, [C.c_char_p, C.POINTER(C.c_int)]),
    "swec_find_dat_file_size": (C.c_int, [C.c_char_p, C.c_char_p, C.POINTER(C.c_int64)]),
    "swec_expected_shard_size": (C.c_int64, [C.c_int64, C.c_int, C.c_int64, C.c_int64]),
    "swec_locate_data": (C.c_int, [C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int,
                                   C.POINTER(Interval), C.c_int]),
    "swec_interval_to_shard": (None, [C.POINTER(Interval), C.c_int64, C.c_int64, C.c_int,
                                      C.POINTER(C.c_int), C.POINTER(C.c_int64)]),
    "swec_alloc_pinned": (C.c_void_p, [C.c_size_t]),
    "swec_alloc_pinned_for_device": (C.c_void_p, [C.c_int, C.c_size_t]),
    "swec_free_pinned": (None, [C.c_void_p]),
    "swec_synth_fill_device": (C.c_int, [C.c_int, C.c_void_p, C.c_uint64, C.c_size_t, C.c_uint64, C.c_void_p]),
    "swec_digest_device": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p]),
}


def library_path() -> str:
    return _LIB_PATH


def lib() -> C.CDLL:
    """Load libswec.so.  Fails loudly if it has not been built — there is no fallback path."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise ImportError(
                f"{_LIB_PATH} is missing: run `python -m seaweedfs_b200.build` (needs nvcc). "
                "seaweedfs_b200 has no CPU fallback.")
        L = C.CDLL(_LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(L, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = L
        import atexit
        atexit.register(L.swec_shutdown)   # before the interpreter starts tearing modules down
    return _lib


def check(status: int) -> None:
    if status != 0:
        raise SwecError(status, lib().swec_last_error().decode(errors="replace"))
