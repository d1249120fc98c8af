/*
 * swec.h — C ABI of the H100-native Reed–Solomon erasure-coding engine for SeaweedFS.
 *
 * This is the drop-in boundary for the RS(10,4) hot path of weed/storage/erasure_coding:
 * a thin cgo file (INTEGRATION.md) binds these entry points in place of
 * github.com/klauspost/reedsolomon (go.mod:50).  Plain pointers and sizes only; every function
 * returns 0 (SWEC_OK) or a negative swec_status, never aborts, never falls back to the CPU: if
 * no CUDA device / kernel image is usable the call fails with SWEC_ERR_NO_DEVICE / SWEC_ERR_CUDA
 * so the caller's cleanup-on-error path runs (weed/server/volume_grpc_erasure_coding.go:78-87).
 *
 * Reference interface each group replaces (paths relative to the SeaweedFS tree):
 *   swec_encoder_new            reedsolomon.New(ds, ps)   weed/storage/erasure_coding/ec_context.go:34-36,
 *                                                          weed/storage/store_ec.go:485
 *   swec_encode                 Encoder.Encode            weed/storage/erasure_coding/ec_encoder.go:265
 *   swec_reconstruct            Encoder.Reconstruct       weed/storage/erasure_coding/ec_encoder.go:360
 *                               Encoder.ReconstructData   weed/storage/store_ec.go:551   (data_only = 1)
 *   swec_verify                 (Rust twin) rs.verify     seaweed-volume/src/storage/erasure_coding/ec_encoder.rs:177-278
 *   swec_write_ec_files         WriteEcFiles / generateEcFiles   ec_encoder.go:61-69,110-128
 *   swec_rebuild_ec_files       RebuildEcFiles / generateMissingEcFiles   ec_encoder.go:74-104,146-200
 *   swec_verify_ec_files        (Rust twin) verify_ec_shards   seaweed-volume/src/storage/erasure_coding/ec_encoder.rs:177-278
 *   swec_locate_ec_damage       what verify_ec_shards cannot tell (ec_encoder.rs:240-258): WHICH shard is wrong
 *   swec_repair_ec_damage       (no counterpart) corrects the located bytes in place instead of rebuilding whole shards
 *   swec_rebuild_ec_files_checked  rebuildEcFiles reading every present shard (ec_encoder.go:342-357), which corrects
 *                               damage in the shards it rebuilds from instead of copying it into the rebuilt ones
 *   swec_reconstruct_batch      batched ReconstructData   weed/storage/store_ec.go:482-560 (one call per interval today)
 *   swec_write_dat_file         WriteDatFile              weed/storage/erasure_coding/ec_decoder.go:176-223
 *   swec_ec_shards_generate     VolumeEcShardsGenerate (file work)   weed/server/volume_grpc_erasure_coding.go:43-146
 *   swec_ec_shards_rebuild      VolumeEcShardsRebuild  (file work)   weed/server/volume_grpc_erasure_coding.go:149-225
 *   swec_ec_shards_to_volume    VolumeEcShardsToVolume (file work)   weed/server/volume_grpc_erasure_coding.go:578-668
 *   swec_ec_shards_to_volume_checked  the same from any k shards, correcting damaged data shards before the .dat is
 *                               written (swec_write_dat_file_checked, swec_decode_data_checked_device)
 *   swec_read_ec_needles        Store.ReadEcShardNeedle (local shards, batched)   weed/storage/store_ec.go:252-355,482-560
 *   swec_check_index_file       idx.CheckIndexFile / EcVolume.ScrubIndex   weed/storage/idx/check.go:36-111
 *   swec_check_needles_device   Needle.ReadBytes on records in HBM   weed/storage/needle/needle_read.go:59-190,
 *                                                          needle_read_tail.go:11-34, crc.go:12-22
 *   swec_ec_volume_*            EcVolume: mount, ReadEcShardNeedle, DeleteNeedleFromEcx, FileAndDeleteCount, ScrubLocal
 *                                                          weed/storage/erasure_coding/ec_volume.go, ec_volume_delete.go, ec_volume_scrub.go
 *   swec_locate_data            LocateData                weed/storage/erasure_coding/ec_locate.go:16-53
 *   swec_expected_shard_size    calculateExpectedShardSize   weed/storage/disk_location_ec.go:428-448
 *
 * Threading: every entry point may be called concurrently from any OS thread (Go schedules
 * gRPC handlers freely; the shell runs up to 10 volumes at once, weed/shell/common.go:11).
 * Calls on ONE encoder handle serialise on its staging buffers; use one handle per goroutine
 * (as the reference does: one reedsolomon.Encoder per file) for parallelism.
 * Ownership: the caller owns every buffer; nothing is retained after a call returns.
 */
#ifndef SWEC_H
#define SWEC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SWEC_MAX_SHARDS 32 /* MaxShardCount, ec_encoder.go:23 */

typedef enum swec_status {
    SWEC_OK = 0,
    SWEC_ERR_INVALID_ARG = -1,     /* bad shard counts, NULL pointers, mismatched sizes        */
    SWEC_ERR_TOO_FEW_SHARDS = -2,  /* fewer than data_shards present (ErrTooFewShards)          */
    SWEC_ERR_CUDA = -3,            /* a CUDA call failed; swec_last_error() has the detail      */
    SWEC_ERR_IO = -4,              /* open/read/write failed; errno text in swec_last_error()   */
    SWEC_ERR_NOMEM = -5,
    SWEC_ERR_SHARD_SIZE = -6,      /* shard files of unequal length ("ec shard size expected…") */
    SWEC_ERR_NO_DEVICE = -7,       /* no usable CUDA device — there is NO CPU fallback          */
    SWEC_ERR_JIT = -8,             /* run-time kernel specialisation failed                     */
    SWEC_ERR_NO_LIVE_NEEDLES = -9, /* ec.decode of a volume whose index has no live entries      */
    SWEC_ERR_NOT_FOUND = -10,      /* needle id not in .ecx (erasure_coding.NotFoundError)       */
    SWEC_ERR_DELETED = -11,        /* needle is tombstoned or journalled (storage.ErrorDeleted)  */
    SWEC_ERR_UNCORRECTABLE = -12   /* checked decode: damage left that cannot be corrected       */
} swec_status;

typedef struct swec_encoder swec_encoder;

/* ---- library ------------------------------------------------------------------------------ */
const char *swec_version(void);
const char *swec_strerror(int status);
const char *swec_last_error(void);            /* thread-local detail of the last failure        */
int swec_device_count(int *count);            /* SWEC_ERR_NO_DEVICE when the driver is absent   */
/* Stop the library's background compiler thread and release the staging rings that file-level calls park
 * for the next call (idempotent).  Embedders whose runtime tears the
 * process down in stages (CPython's Py_Finalize) call this from their own exit hook; the library
 * also registers it with atexit().  Everything keeps working afterwards, without background JIT. */
void swec_shutdown(void);
/* Device ids interleaved over the host's NUMA nodes (0,4,1,5,… on a 2-socket, 8-GPU box): the first n entries are the
 * n GPUs a process should use for n concurrent host-fed volumes — one socket cannot feed four GPUs at full PCIe rate.
 * This is the order swecPickDevice (INTEGRATION.md) walks; weed/shell/command_ec_encode.go:302-315 runs the volumes.   */
int swec_device_spread_order(int *order, int capacity, int *count);
uint64_t swec_kernel_launches(void);          /* kernels this process has launched (all devices) */
/* Tuning: "enc_threads" {128,256,512}, "enc_unroll" {1,2}, "ctas_per_sm" (0 = auto),
 * "stage_chunk" (bytes per shard per staging slot), "stage_slots" {2..16} (slots in flight per staging ring, for
 * host-buffer and file-level calls alike; SWEC_STAGE_SLOTS sets it at load), "host_pieces" (a host-buffer call is cut
 * into at least this many pipelined pieces), "host_min_chunk" (but none smaller than this many bytes per shard), "jit" {0,1},
 * "jit_min_bytes" (streams at least this long compile their kernel inline, shorter ones in the
 * background), "power_mode" {0 = auto by the device's recent kernel time — for a GPU that sits on its power cap under
 * back-to-back launches, where the variant with fewer instructions can be the faster one; 1 = always the boost-clock
 * kernel variant (default: an H100 SXM at 700 W keeps its clock and runs it ~4 % faster when sustained); 2 = always the
 * low-power one}, "host_zero_copy" {0,1,2 = auto:
 * host-buffer calls of at most "host_zero_copy_max" bytes per shard run the kernel directly on the (mapped, pinned) host
 * memory over PCIe instead of staging through HBM}, "file_direct_io" {bit 0: O_DIRECT reads, bit 1: O_DIRECT writes in
 * the file-level entry points}.  Measurement knobs: "xt_variant" {0..3} (instruction mix of run-time specialised kernels,
 * device_common.cuh), "use_aot" {0,1} (0: RS(10,4) encode is specialised at run time like any matrix), "jit_share_powers"
 * {0,1} (1: run-time specialised kernels are generated with shared power chains — fewer multiply-by-2 steps; bytes
 * checked on the GPU, speed not yet measured, hence off).  Changing any of enc_threads, enc_unroll, xt_variant,
 * power_mode or jit_share_powers makes later calls use (and if needed compile) the kernel of the new setting. */
int swec_set_option(const char *name, long value);
/* Diagnostics: generate and NVRTC-compile (sm_90a) the specialised kernel for an r×k matrix without
 * loading it — needs no GPU.  Reports the cubin size and the generator's instruction statistics.  */
int swec_debug_jit_compile(int r, int k, const uint8_t *rows, size_t *cubin_bytes, int *xtime_steps,
                           int *xor_ops);
/* Diagnostics of "power_mode" auto: `heat_ms` = estimated Horner-kernel milliseconds the device ran during the last
 * second (exponentially decayed; continuous encoding tends to 1000), `low_power` = the variant the next launch takes
 * (1 once heat_ms exceeds 450).  device < 0: the calling thread's current device.                                  */
int swec_debug_power_state(int device, double *heat_ms, int *low_power);
/* The decode-kernel cache (GPU analogue of the decode-matrix LRU, rse/src/core.rs:25,700-734), three tiers:
 * `aot_matrices` reconstruct matrices compiled with the library (every single-shard loss of RS(10,4) and shards 0-3
 * lost: no compile, no NVRTC, any stream length); an on-disk cubin cache shared by every process
 * ($SWEC_CACHE_DIR, else $XDG_CACHE_HOME/swec, else ~/.cache/swec; SWEC_NO_DISK_CACHE=1 disables; a directory that does
 * not belong to the calling user or that group/others can write to is not trusted with executable code and is ignored) whose hits are
 * counted in `disk_cache_hits`; NVRTC for patterns never seen before (`nvrtc_compiles`).  `aot_launches` = launches of
 * the compiled-in reconstruct kernels by this process.  Any pointer may be NULL. */
int swec_jit_stats(uint64_t *nvrtc_compiles, uint64_t *disk_cache_hits, int *aot_matrices,
                   uint64_t *aot_launches);

/* ---- encoder = reedsolomon.New(dataShards, parityShards) ----------------------------------- */
/* device < 0: host-side object only (matrix queries); compute calls then fail with NO_DEVICE.  */
int swec_encoder_new(int data_shards, int parity_shards, int device, swec_encoder **out);
void swec_encoder_free(swec_encoder *enc);
/* (k+m)×k generator matrix, row-major: identity on top, parity rows below.                     */
int swec_encoder_matrix(const swec_encoder *enc, uint8_t *out);
/* The fused matrix Reconstruct would apply for a presence mask: inputs[k] (shard ids read),
 * outputs[*n_outputs] (shard ids produced), rows[*n_outputs * k].                              */
int swec_reconstruct_matrix(const swec_encoder *enc, const uint8_t *present, int data_only,
                            int *inputs, int *outputs, int *n_outputs, uint8_t *rows);

/* ---- Encoder.Encode / Reconstruct / ReconstructData on HOST buffers ------------------------- */
/* shards[0..k) are read, shards[k..k+m) are overwritten; all shard_len bytes, shard_len > 0.   */
int swec_encode(swec_encoder *enc, uint8_t *const *shards, size_t shard_len);
/* present[i] != 0 ⇔ shards[i] holds data.  Missing shards must point at shard_len writable
 * bytes (the cgo shim allocates them, as klauspost does for nil slices).  data_only = 1 fills
 * only indices < k (ReconstructData).  All present ⇒ no-op; fewer than k ⇒ TOO_FEW_SHARDS.     */
int swec_reconstruct(swec_encoder *enc, uint8_t *const *shards, const uint8_t *present,
                     size_t shard_len, int data_only);
/* Many ReconstructData/Reconstruct calls at once — the batched form of the degraded-read path
 * (store_ec.go:482-560 issues one tiny call per needle interval).  Items that share a presence
 * mask are packed into common launches; results are identical to calling swec_reconstruct on each. */
typedef struct swec_reconstruct_item {
    uint8_t *const *shards;   /* k+m pointers, as for swec_reconstruct */
    const uint8_t *present;   /* k+m flags */
    size_t shard_len;
    int data_only;
} swec_reconstruct_item;
int swec_reconstruct_batch(swec_encoder *enc, const swec_reconstruct_item *items, int n_items);
/* One call, several GPUs: the byte-column range [0, shard_len) is cut into n_encs contiguous pieces and
 * piece g goes through encs[g] (one handle per GPU, created with swec_encoder_new(k, m, device_g)), all
 * pieces concurrently, each over its own GPU's PCIe link.  Columns are independent, so the result is
 * byte-identical to swec_encode / swec_reconstruct on one handle; there is no inter-GPU traffic.  This
 * is the second axis of independence of SURVEY §8e (the first — whole volumes round-robin over GPUs —
 * needs no API: give each concurrent volume a handle on another device).                            */
int swec_encode_multi(swec_encoder *const *encs, int n_encs, uint8_t *const *shards, size_t shard_len);
int swec_reconstruct_multi(swec_encoder *const *encs, int n_encs, uint8_t *const *shards,
                           const uint8_t *present, size_t shard_len, int data_only);
/* n_shards pinned buffers of shard_len bytes laid out FOR such a call: byte range g of every shard is bound to the
 * NUMA node of encs[g]'s GPU (the split rule is shared), so each GPU DMAs from its own socket.  One allocation:
 * release it with swec_free_pinned(shards[0]).                                                                */
int swec_alloc_pinned_shards(swec_encoder *const *encs, int n_encs, int n_shards, size_t shard_len,
                             uint8_t **shards);
/* *ok = 1 iff the parity shards match the data shards.                                         */
int swec_verify(swec_encoder *enc, uint8_t *const *shards, size_t shard_len, int *ok);

/* ---- the same on DEVICE buffers, asynchronous on `stream` (a cudaStream_t; NULL = the CUDA
 *      default stream).  Buffers must stay valid until the stream reaches this point. --------- */
int swec_encode_device(swec_encoder *enc, const void *const *data, void *const *parity,
                       size_t shard_len, void *stream);
int swec_reconstruct_device(swec_encoder *enc, void *const *shards, const uint8_t *present,
                            size_t shard_len, int data_only, void *stream);
/* The primitive underneath: out[p][x] = XOR_i rows[p*k+i] ⊗ in[i][x] for any r×k matrix over
 * GF(2^8)/0x11D (k ≤ 32) — what code_some_slices does (reed-solomon-erasure core.rs:484-512).    */
int swec_apply_device(swec_encoder *enc, int r, int k, const uint8_t *rows, const void *const *in,
                      void *const *out, size_t shard_len, void *stream);
/* A whole volume image resident in HBM → parity shard images, following the two-tier striping
 * of encodeDatFile (ec_encoder.go:280-321): rows of k large blocks while ≥ k*large bytes
 * remain, then rows of k small blocks, the last one zero-padded.  parity[p] receives
 * swec_expected_shard_size() bytes.  Data shards are views of the image and are not copied.    */
int swec_encode_volume_device(swec_encoder *enc, const void *dat, int64_t dat_size,
                              int64_t large_block, int64_t small_block, void *const *parity,
                              void *stream);
/* Gather data shard `shard_id` of the image into a contiguous shard buffer (what .ecNN holds).  */
int swec_extract_data_shard_device(swec_encoder *enc, const void *dat, int64_t dat_size,
                                   int64_t large_block, int64_t small_block, int shard_id,
                                   void *shard_out, void *stream);
/* WriteDatFile on device memory (weed/storage/erasure_coding/ec_decoder.go:176-223, the body of ec.decode): the k data
 * shards, each swec_expected_shard_size() bytes in HBM (as read from .ec00-.ec09, or as swec_reconstruct_device just
 * rebuilt them), are un-striped into the dat_size bytes of the volume image — rows of k large blocks while at least one
 * full large row remains, then rows of k small blocks, the zero padding of the last row dropped.  Exact inverse of
 * swec_extract_data_shard_device; k strided device-to-device copies per region, asynchronous on `stream`.           */
int swec_write_dat_device(swec_encoder *enc, const void *const *data_shards, int64_t dat_size,
                          int64_t large_block, int64_t small_block, void *dat_out, void *stream);
int swec_stream_synchronize(swec_encoder *enc, void *stream);

/* ---- file level: .dat → .ec00…, missing .ecNN ← the others, .ec00–.ec09 → .dat -------------- */
/* WriteEcFiles(baseFileName): RS(10,4), 1 GiB / 1 MiB blocks.                                   */
int swec_write_ec_files(const char *base_file_name, int device);
/* generateEcFiles(base, bufferSize, large, small, ctx).  buffer_size only has to divide both
 * block sizes (the reference Fatalf's otherwise); results do not depend on it.                  */
int swec_generate_ec_files(const char *base_file_name, int64_t buffer_size, int64_t large_block,
                           int64_t small_block, int data_shards, int parity_shards, int device);
/* RebuildEcFiles(base, additionalDirs...).  data_shards = 0 ⇒ take the ratio from base.vif
 * (ecShardConfig) when valid, else 10+4 (ec_encoder.go:76-95).  rebuilt[] (≥ SWEC_MAX_SHARDS
 * entries) receives the generated shard ids.                                                    */
int swec_rebuild_ec_files(const char *base_file_name, const char *const *additional_dirs,
                          int n_additional_dirs, int data_shards, int parity_shards, int device,
                          uint32_t *rebuilt, int *n_rebuilt);
/* Scrub: re-encode .ec00–.ec(k-1) on the GPU and compare with the parity shards on disk (the Rust
 * twin's verify_ec_shards, seaweed-volume/src/storage/erasure_coding/ec_encoder.rs:177-278; the Go
 * scrub never checks parity, ec_volume_scrub.go:27-118).  mismatched_vectors[p] (m entries, may be
 * NULL) = number of differing 16-byte vectors in parity shard p, the partial last vector of a length
 * that is not a multiple of 16 counting as one; *ok = 1 iff all are zero.                          */
int swec_verify_ec_files(const char *base_file_name, const char *const *additional_dirs,
                         int n_additional_dirs, int data_shards, int parity_shards, int device,
                         uint64_t *mismatched_vectors, int *ok);

/* ---- locate the wrong shard when parity does not match ----------------------------------------------------------
 * Per byte column x, computed parity XOR stored parity is the syndrome s = [P | I]·e of the column's error pattern e.
 * A GPU kernel decodes every non-zero syndrome within `radius` wrong shards and blames those shards.  RS(k,m) has
 * minimum distance m+1, so radius-t decoding (t = 1 or 2, 2t <= m) guarantees, per column:
 *   - at most t wrong shards: exactly those shards are blamed;
 *   - more than t but at most m-t wrong shards: the column is counted as uncorrectable and no shard is blamed;
 *   - more than m-t wrong shards: the column may be blamed on the wrong shards.  That is the limit of the code.
 * For RS(10,4), radius 1 (the default) is always right, or says uncorrectable, for up to 3 damaged shards per column;
 * radius 2 locates overlapping damage in 2 shards but may misattribute 3.  swec_repair_ec_damage (below) corrects the
 * located bytes in place; where it leaves uncorrectable columns, or a shard file is missing, the remedy is to delete the
 * blamed shard files and run swec_rebuild_ec_files.  The reference cannot do this: verify_ec_shards
 * (seaweed-volume/src/storage/erasure_coding/ec_encoder.rs:240-258) marks every mismatching PARITY shard as broken, so
 * one damaged data shard gets all m parity shards reported (and rebuilding those bakes the damage in), and the Go scrub
 * never checks parity (ec_volume_scrub.go:25).                                                                        */
typedef struct swec_damage_report {
    uint64_t columns;                        /* byte columns checked (= shard length)                         */
    uint64_t damaged_columns;                /* columns with a non-zero syndrome                              */
    uint64_t uncorrectable_columns;          /* ... that no pattern of <= radius shards explains              */
    int64_t first_uncorrectable, last_uncorrectable;  /* shard offsets; -1 when none                        */
    uint64_t shard_bytes[SWEC_MAX_SHARDS];   /* bytes of shard i located as wrong                             */
    int64_t shard_first[SWEC_MAX_SHARDS], shard_last[SWEC_MAX_SHARDS];  /* -1 when none                      */
} swec_damage_report;
typedef struct swec_damage_range {
    int32_t shard_id; /* -1 = uncorrectable columns                                                          */
    int32_t reserved;
    int64_t offset;   /* 4 KiB-aligned shard offset                                                          */
    int64_t length;   /* whole 4 KiB pages, the last one clipped to the shard length                         */
} swec_damage_range;
/* Both calls: ranges are the maximal runs of consecutive 4 KiB pages holding a blamed column, per shard (ascending id,
 * then offset), followed by the runs holding uncorrectable columns.  *n_ranges (may be NULL) = how many there are; only
 * the first ranges_cap are written.  radius must be 1 or 2, radius 1 needs m >= 2 and radius 2 needs m >= 4; report
 * must not be NULL and ranges_cap not negative (SWEC_ERR_INVALID_ARG otherwise).
 * File level: the shard lookup, ratio rule (data_shards = 0: from base.vif) and errors of swec_verify_ec_files, the same
 * file pipeline, and the locate kernel in place of the compare.  Every file check happens before any device work; an
 * encoder without a device fails with SWEC_ERR_NO_DEVICE.  *ok = 1 iff no column has a non-zero syndrome.           */
int swec_locate_ec_damage(const char *base_file_name, const char *const *additional_dirs, int n_additional_dirs,
                          int data_shards, int parity_shards, int device, int radius, swec_damage_report *report,
                          swec_damage_range *ranges, int ranges_cap, int *n_ranges, int *ok);
/* Device level: shards[k+m] in HBM, shard_len bytes each.  The parity is recomputed with the encode kernel into scratch
 * of at most 256 MiB per parity shard at a time (no run-time compile for RS(10,4)); synchronises `stream`.           */
int swec_locate_damage_device(swec_encoder *enc, const void *const *shards, size_t shard_len, int radius,
                              swec_damage_report *report, swec_damage_range *ranges, int ranges_cap,
                              int *n_ranges, void *stream);
/* ---- repair in place: the locate calls, which also write the corrections --------------------------------------------
 * Same arguments, argument rules and report as the locate calls; the report is the one they return for the same input
 * before the call, so shard_bytes[i] = the bytes corrected in shard i.
 *   - In every column where at most `radius` shards are blamed, the blamed bytes are replaced by the decoded values, and
 *     the column is a codeword again.  Uncorrectable columns are left byte for byte as they were.
 *   - The guarantee above carries over unchanged, and so does its limit: a column with more than m-t wrong shards can be
 *     MISCORRECTED, that is rewritten into a different codeword.  For RS(10,4), radius 1 never miscorrects a column
 *     with up to 3 wrong shards; radius 2 can miscorrect a column with 3 or more.  Radius 1 is the default of every
 *     binding; take radius 2 only for damage known to overlap in at most 2 shards.
 *   - A clean set is never written to, so a second call on a repaired set reports damaged_columns == 0.
 * File level: pass 1 is swec_locate_ec_damage (same shard lookup, ratio rule, errors and kernel launches), and a set
 * without damage is left there, never opened for writing.  A missing shard is SWEC_ERR_TOO_FEW_SHARDS (rebuild first)
 * and unequal lengths SWEC_ERR_SHARD_SIZE, both before any device work and before anything is opened for writing.
 * Pass 2 reads again only the 4 KiB pages pass 1 flagged, corrects them on the GPU, and pwrites each blamed shard's own
 * flagged pages back to the file where the shard was found (base directory or an additional dir), with O_DIRECT when
 * "file_direct_io" bit 1 is set; every modified file is fdatasync'ed before the call returns.  *ok = 1 iff no
 * uncorrectable column remains.  As for rebuild, nobody else may write the shard files during the call.  Each byte is
 * written once, old or corrected, so a repair cut short by a crash leaves every column as it was, corrected, or (at
 * radius 2) corrected in one of its two shards, which is still within the radius: running the call again finishes it.
 * Device level: the shards in HBM are corrected the same way, each 256 MiB piece after its parity was recomputed, in
 * stream order; synchronises `stream`.                                                                               */
int swec_repair_ec_damage(const char *base_file_name, const char *const *additional_dirs, int n_additional_dirs,
                          int data_shards, int parity_shards, int device, int radius, swec_damage_report *report,
                          swec_damage_range *ranges, int ranges_cap, int *n_ranges, int *ok);
int swec_correct_damage_device(swec_encoder *enc, void *const *shards, size_t shard_len, int radius,
                               swec_damage_report *report, swec_damage_range *ranges, int ranges_cap,
                               int *n_ranges, void *stream);
/* ---- checked rebuild: errors and erasures ---------------------------------------------------------------------------
 * swec_rebuild_ec_files reads only the first k present shards, so a wrong byte in one of them goes into every shard it
 * rebuilds.  The checked rebuild reads every present shard.  The first k present shards are the information set; the
 * other c = m - f present shards (f = missing shards) are its check shards, re-encoded and compared, and the damage the
 * syndrome locates in the information set is taken out of the rebuilt bytes.  The present shards form a code of
 * distance c+1, and the radius used is t = min(radius, floor(c/2)); radius may be 0, 1 or 2.  Per column:
 *   - at most t wrong present shards: exactly those shards are blamed, and the rebuilt bytes are the true ones;
 *   - t+1 .. c-t wrong present shards: the column is counted as uncorrectable, nothing is blamed, and its rebuilt bytes
 *     are exactly what swec_rebuild_ec_files writes;
 *   - more than c-t wrong present shards: the blame and the rebuilt bytes can both be wrong.  That includes a column in
 *     which only check shards are wrong, which plain rebuild would have rebuilt right;
 *   - radius 0 (detect only): a column with 1 .. c wrong present shards is always counted as uncorrectable and rebuilt
 *     exactly as plain rebuild does.  Take it when no guess is wanted, notably when c is 2 or 3.
 * For RS(10,4) at radius 1: with 1 shard lost (c = 3), 1 wrong present shard is corrected and 2 are reported; with 2
 * lost (c = 2), 1 is corrected and 2 can be wrong (radius 0 reports them instead); with 3 lost (c = 1), 1 is reported;
 * with 4 lost nothing can be checked.  With nothing lost (c = m) the report is the one of swec_locate_ec_damage.
 * Present shards are never written, neither the files nor the device buffers.  To fix them, run swec_repair_ec_damage
 * (or swec_correct_damage_device) on the completed set afterwards: with every rebuilt column right, a column with one
 * damaged present shard is within radius 1 of the full code.
 * The report and ranges are those of the locate calls, over the present shards (a missing shard is never blamed);
 * with c = 0 the report has columns = 0 and no ranges.  Argument rules: report not NULL, ranges_cap not negative,
 * ranges not NULL when ranges_cap > 0, radius 0, 1 or 2 (SWEC_ERR_INVALID_ARG otherwise, before anything else).
 * File level: the arguments, ratio rule, shard lookup, errors and texts of swec_rebuild_ec_files, in its order (too few
 * shards before any output exists; the outputs created, then the lengths compared; on any failure no ids and no
 * output file left).  rebuilt[] receives the rebuilt ids (none when nothing is missing; then nothing is written).  The
 * rebuilt files are written even where uncorrectable columns remain; the ranges say where.  *ok = 1 iff c >= 1 and no
 * column is uncorrectable.
 * Device level: the argument rules of swec_reconstruct_device (a shard to rebuild needs a buffer, fewer than k present
 * is SWEC_ERR_TOO_FEW_SHARDS) plus the ones above.  The check shards are re-encoded into scratch of at most 256 MiB per
 * shard at a time; synchronises `stream`.                                                                             */
int swec_rebuild_ec_files_checked(const char *base_file_name, const char *const *additional_dirs, int n_additional_dirs,
                                  int data_shards, int parity_shards, int device, int radius,
                                  uint32_t *rebuilt, int *n_rebuilt, swec_damage_report *report,
                                  swec_damage_range *ranges, int ranges_cap, int *n_ranges, int *ok);
int swec_reconstruct_checked_device(swec_encoder *enc, void *const *shards, const uint8_t *present, size_t shard_len,
                                    int radius, swec_damage_report *report, swec_damage_range *ranges, int ranges_cap,
                                    int *n_ranges, void *stream);
int swec_write_dat_file(const char *base_file_name, int64_t dat_file_size,
                        const char *const *shard_file_names, int data_shards,
                        int64_t large_block, int64_t small_block);
/* ---- checked decode: errors and erasures before the parity is dropped -----------------------------------------------
 * ec.decode deletes every shard, parity included, once the .dat is written (weed/shell/command_ec_decode.go:156-181),
 * so it is the last point at which damage in the data shards can be corrected.  swec_write_dat_file copies the data
 * shards byte for byte and needs all of them.  The checked decode needs any k of the k+m shards.  It decodes like the
 * checked rebuild above: the first k present shards are the information set, the other c = (present shards) - k are
 * its check shards (always parity shards), and the radius used is t = min(radius, floor(c/2)), radius 0, 1 or 2.
 * Unlike the checked rebuild, it also corrects the damage located in present data shards, so per column:
 *   - at most t wrong present shards: every data byte of the column is the true one, present or rebuilt;
 *   - t+1 .. c-t wrong present shards: the column is counted as uncorrectable, and its data bytes are exactly what
 *     swec_reconstruct_device(data_only = 1) gives from the shards as found;
 *   - more than c-t wrong present shards: the data bytes can be wrong (the limit of the code);
 *   - radius 0: every damaged column is uncorrectable.
 * Only missing data shards are rebuilt; a missing parity shard is neither computed nor needed.  Present parity is only
 * read.  The report and ranges are those of the checked rebuild for the same shards; with c = 0 the report has
 * columns = 0 and no ranges.  Argument rules: those of swec_reconstruct_checked_device (SWEC_ERR_INVALID_ARG first).
 * Device level: shards[k+m] in HBM, shard_len bytes each.  Every data shard needs a buffer: present ones are corrected in
 * place, missing ones rebuilt.  A missing parity shard may be NULL.  Fewer than k present is SWEC_ERR_TOO_FEW_SHARDS.
 * The check shards are re-encoded into scratch of at most 256 MiB per shard at a time; synchronises `stream`.  With
 * c = 0 it is swec_reconstruct_device(data_only = 1).
 * File level: swec_write_dat_file_checked is swec_write_dat_file from shard_file_names[k+m] (NULL = missing): the same
 * copy plan and the same .dat bytes, as if written from the corrected data shards.  The columns decoded are those the
 * plan reads from shard 0, [0, columns).  Before any device work and before the .dat is created, in this order: fewer
 * than k shards present is SWEC_ERR_TOO_FEW_SHARDS, present shards of unequal length SWEC_ERR_SHARD_SIZE, and shards
 * shorter than the plan needs SWEC_ERR_IO (the short read of the plain call).  Shard files are never opened for writing.
 * If any column is left uncorrectable the call fails with SWEC_ERR_UNCORRECTABLE and removes the .dat, with the report
 * and ranges filled in: a caller that then keeps the EC shards loses nothing.  Radius 0 therefore decodes only a set
 * in which every checked column is clean.  On any other failure no .dat is left either.  *ok = 1 iff c >= 1 and no
 * column is uncorrectable.  With every data shard present and no parity shard (c = 0, nothing missing) there is
 * nothing to check or rebuild: the call is swec_write_dat_file, with no GPU work, columns = 0 and *ok = 0.
 * swec_ec_shards_to_volume_checked is swec_ec_shards_to_volume with this call in place of swec_write_dat_file, and any k
 * shards instead of all k data shards: the ratio from .vif, the shards looked up in data_base's directory then in
 * additional_dirs (fewer than k found: SWEC_ERR_TOO_FEW_SHARDS), the .ecj folded into .ecx, SWEC_ERR_NO_LIVE_NEEDLES,
 * FindDatFileSize, the .dat, the .idx.  FindDatFileSize takes the needle version from the .ec00 superblock, or from
 * .vif's version when .ec00 is missing; with neither the call fails with SWEC_ERR_TOO_FEW_SHARDS before anything is
 * written.  On SWEC_ERR_UNCORRECTABLE neither .dat nor .idx is left.                                                */
int swec_decode_data_checked_device(swec_encoder *enc, void *const *shards, const uint8_t *present, size_t shard_len,
                                    int radius, swec_damage_report *report, swec_damage_range *ranges, int ranges_cap,
                                    int *n_ranges, void *stream);
int swec_write_dat_file_checked(const char *base_file_name, int64_t dat_file_size, const char *const *shard_file_names,
                                int data_shards, int parity_shards, int64_t large_block, int64_t small_block,
                                int device, int radius, swec_damage_report *report, swec_damage_range *ranges,
                                int ranges_cap, int *n_ranges, int *ok);

/* ---- whole-volume operations: what the three EC gRPC handlers do to files, in their order --------- */
/* VolumeEcShardsGenerate: ratio from data_base.vif when valid else 10+4; index_base.idx → .ecx FIRST;
 * snapshot the .dat size; .dat → .ec00… on the GPU (256 KiB / 1 GiB / 1 MiB); write data_base.vif
 * {version, datFileSize, expireAtSec, ecShardConfig}.  On any error the shard files and the .ecx are
 * removed (the handler's deferred cleanup).  index_base NULL/"" = data_base.  needle_version 0 = read
 * it from the .dat superblock.                                                                      */
int swec_ec_shards_generate(const char *data_base_file_name, const char *index_base_file_name,
                            uint32_t needle_version, uint64_t expire_at_sec, int device);
/* VolumeEcShardsRebuild: RebuildEcFiles(data_base, additional_dirs...) then RebuildEcxFile(index_base,
 * or data_base when index_base has no .ecx).                                                        */
int swec_ec_shards_rebuild(const char *data_base_file_name, const char *index_base_file_name,
                           const char *const *additional_dirs, int n_additional_dirs, int device,
                           uint32_t *rebuilt, int *n_rebuilt);
/* VolumeEcShardsToVolume (ec.decode): needs all data shards (data_base's directory, then
 * additional_dirs); RebuildEcxFile → HasLiveNeedles (SWEC_ERR_NO_LIVE_NEEDLES when none) →
 * FindDatFileSize → WriteDatFile → WriteIdxFileFromEcIndex.  No GPU work.  *dat_file_size may be NULL. */
int swec_ec_shards_to_volume(const char *data_base_file_name, const char *index_base_file_name,
                             const char *const *additional_dirs, int n_additional_dirs,
                             int64_t *dat_file_size);
/* The same from any k of the k+m shards, correcting damaged data shards on the GPU first (see the checked decode
 * above).  *dat_file_size may be NULL.                                                                              */
int swec_ec_shards_to_volume_checked(const char *data_base_file_name, const char *index_base_file_name,
                                     const char *const *additional_dirs, int n_additional_dirs, int device,
                                     int radius, int64_t *dat_file_size, swec_damage_report *report,
                                     swec_damage_range *ranges, int ranges_cap, int *n_ranges, int *ok);

/* Store.ReadEcShardNeedle for MANY needles of one EC volume whose shard files are local (data_base's
 * directory, then additional_dirs) — weed/storage/store_ec.go:252-355,482-560: find each needle in .ecx
 * (journalled ids read as deleted), LocateData its record through the two-tier layout (shard size from
 * .vif's datFileSize, else shard file size - 1), pread every interval whose shard file is present and
 * recover the others from the same interval of all remaining shards with ReconstructData.  All
 * recoveries of the call go to the GPU as ONE swec_reconstruct_batch; with every needed shard present the
 * call does no GPU work at all.  buf receives the raw record bytes exactly as the reference's `bytes`
 * (which over-reads: GetActualSize is applied twice, ec_volume.go:395,414); parsing them is the storage
 * engine's business.  Per-needle outcome in status: SWEC_OK, SWEC_ERR_NOT_FOUND, SWEC_ERR_DELETED,
 * SWEC_ERR_TOO_FEW_SHARDS, or SWEC_ERR_INVALID_ARG when capacity < the n_bytes reported back.        */
typedef struct swec_needle_read {
    uint64_t needle_id;            /* in  */
    uint8_t *buf;                  /* in  */
    size_t capacity;               /* in  */
    int64_t offset;                /* out: byte offset of the record in the .dat                  */
    int32_t size;                  /* out: Size field of the index entry (negative = deleted)      */
    int32_t status;                /* out */
    size_t n_bytes;                /* out: bytes stored in buf (or needed, on SWEC_ERR_INVALID_ARG) */
    int32_t n_recovered_intervals; /* out: intervals that were reconstructed rather than read      */
    int32_t reserved;
} swec_needle_read;
int swec_read_ec_needles(const char *data_base_file_name, const char *index_base_file_name,
                         const char *const *additional_dirs, int n_additional_dirs,
                         swec_needle_read *reads, int n_reads, int device);
/* The same on a MOUNTED volume — the twin of the long-lived EcVolume (ec_volume.go:36-160): open once
 * (ratio / needle version / datFileSize from .vif, shard files opened, .ecx loaded, .ecj re-read when it
 * grows), read many times; the encoder behind the recoveries, its staging ring and its specialised kernels
 * live as long as the handle.  Calls on one handle serialise.  swec_read_ec_needles = open + read + close. */
typedef struct swec_ec_volume swec_ec_volume;
int swec_ec_volume_open(const char *data_base_file_name, const char *index_base_file_name,
                        const char *const *additional_dirs, int n_additional_dirs, int device,
                        swec_ec_volume **out);
int swec_ec_volume_read_needles(swec_ec_volume *vol, swec_needle_read *reads, int n_reads);
/* EcVolume.DeleteNeedleFromEcx (ec_volume_delete.go:28-93): append the id to the .ecj journal (fsync'ed
 * before it becomes visible to reads); unknown, tombstoned or already journalled ids are not errors.  */
int swec_ec_volume_delete_needle(swec_ec_volume *vol, uint64_t needle_id);
/* EcVolume.ScrubLocal (ec_volume_scrub.go:27-118) without the needle parse: ScrubIndex (swec_check_index_file on the
 * .ecx), then every live entry is located and each of its chunks read from the local shard that should hold it.
 * broken_shards[SWEC_MAX_SHARDS] receives the ids (ascending) of shards that were too short or unreadable for some
 * chunk; findings are newline-separated in errors[], worded like the reference.  Parity is checked by
 * swec_verify_ec_files; swec_ec_volume_scrub_needles adds the needle parse.  No GPU work.                     */
int swec_ec_volume_scrub_local(swec_ec_volume *vol, int64_t *entries, uint32_t *broken_shards, int *n_broken,
                               char *errors, size_t errors_cap, int *n_errors);
/* The whole EcVolume.ScrubLocal: the walk of swec_ec_volume_scrub_local, and every record whose chunks are all local
 * is checked like Needle.ReadBytes (size, layout, CRC32-C) on the GPU of the volume's device.  Records are read
 * straight into pinned staging slots and checked a slot at a time while the walk fills the next slot.  A failed
 * record adds "needle <id> on volume <volume_id>: <err>" after the findings of the records walked before it, with
 * <err> as ReadBytes words it ("size mismatch", "index out of range N: needle data corrupted", "invalid CRC for
 * needle <hex id> (got %08x, want %08x), data on disk corrupted: needle data corrupted").  A walk with nothing to
 * check does no GPU work; otherwise a volume opened with device < 0 fails with SWEC_ERR_NO_DEVICE.           */
int swec_ec_volume_scrub_needles(swec_ec_volume *vol, uint32_t volume_id, int64_t *entries, uint32_t *broken_shards,
                                 int *n_broken, char *errors, size_t errors_cap, int *n_errors);
/* What mounting derived (NewEcVolume, ec_volume.go:114-154,399-417): EC ratio and needle version from .vif (defaults
 * 10+4, version 3), the shard size LocateData works with, and a bit per shard file found locally.  Any out pointer
 * may be NULL.                                                                                                 */
int swec_ec_volume_info(swec_ec_volume *vol, int *data_shards, int *parity_shards, int *needle_version,
                        int64_t *shard_dat_size, uint32_t *local_shard_bits);
/* EcVolume.FileAndDeleteCount (ec_volume.go:330-349): .ecx entries, distinct journalled deletions.      */
int swec_ec_volume_counts(swec_ec_volume *vol, uint64_t *file_count, uint64_t *delete_count);
void swec_ec_volume_close(swec_ec_volume *vol);

/* ---- needle records on the GPU: Needle.ReadBytes (weed/storage/needle/needle_read.go:59-190) ------------------ */
typedef enum swec_needle_status {
    SWEC_NEEDLE_OK = 0,
    SWEC_NEEDLE_SIZE_MISMATCH = 1,  /* header Size != index Size (ErrorSizeMismatch)                       */
    SWEC_NEEDLE_OUT_OF_RANGE = 2,   /* DataSize or an optional field overruns the body; range_index 1..7  */
    SWEC_NEEDLE_BAD_CRC = 3,        /* CRC32-C of Data != the stored checksum                             */
    SWEC_NEEDLE_OUTSIDE_IMAGE = 4   /* the record does not fit inside the image: not read at all          */
} swec_needle_status;
typedef struct swec_needle_check {
    uint64_t needle_id;   /* in  (reported back only)                                                       */
    int64_t offset;       /* in  byte offset of the record in the image                                     */
    int32_t size;         /* in  Size of the index entry                                                    */
    int32_t status;       /* out swec_needle_status                                                         */
    int32_t range_index;  /* out 1..7 with SWEC_NEEDLE_OUT_OF_RANGE, else 0                                 */
    uint32_t data_size;   /* out bytes of Data (the whole body in version 1)                                */
    uint32_t crc_got;     /* out CRC32-C (Castagnoli) of Data, as Go's crc32.Update(0, Castagnoli table, Data) */
    uint32_t crc_want;    /* out the big-endian checksum stored after the body                              */
    int32_t legacy_crc;   /* out 1 when crc_want is the pre-3.09 CRC.Value() form of crc_got (crc.go:25-27):  */
                          /*     ReadBytes still reports the record, but it is old, not corrupt             */
    int32_t reserved;
} swec_needle_check;
/* Check n records of a volume image (.dat bytes, superblock included) resident in HBM, each the way
 * Needle.ReadBytes(record, 0, size, version) does, stopping at a record's first failure.  `dat` is a device pointer;
 * checks[] is host memory.  A record that does not end inside dat_size is SWEC_NEEDLE_OUTSIDE_IMAGE and is never
 * read.  Synchronises `stream` (a cudaStream_t; NULL = the default stream).                                        */
int swec_check_needles_device(int device, const void *dat, int64_t dat_size, int needle_version,
                              swec_needle_check *checks, int n, void *stream);

/* ---- index files either side of the path (host only, no GPU) ---------------------------------- */
/* WriteSortedFileFromIdx(base, ext): base.idx → base+ext (".ecx"), live entries sorted by needle id
 * (ec_encoder.go:31-58).  Call it BEFORE writing shards, as VolumeEcShardsGenerate does.          */
int swec_write_sorted_file_from_idx(const char *base_file_name, const char *ext);
/* RebuildEcxFile: fold the .ecj deletion journal into .ecx, then remove .ecj
 * (ec_volume_delete.go:95-142).                                                                  */
int swec_rebuild_ecx_file(const char *base_file_name);
/* WriteIdxFileFromEcIndex: .ecx (+ one tombstone per .ecj id) → .idx (ec_decoder.go:35-60).       */
int swec_write_idx_file_from_ec_index(const char *base_file_name);
/* idx.CheckIndexFile (weed/storage/idx/check.go:36-111) = EcVolume.ScrubIndex on an .ecx (or an .idx): entries
 * processed, and one message per finding — overlapping neighbours in (offset, size) order, a file that is not a whole
 * number of entries — newline-separated into errors[errors_cap] (may be NULL), worded like the reference.        */
int swec_check_index_file(const char *path, int needle_version, int64_t *entries, char *errors,
                          size_t errors_cap, int *n_errors);
/* HasLiveNeedles / FindDatFileSize (ec_decoder.go:23-33, 65-92).                                  */
int swec_has_live_needles(const char *index_base_file_name, int *has_live);
int swec_find_dat_file_size(const char *data_base_file_name, const char *index_base_file_name,
                            int64_t *dat_size);

/* ---- layout arithmetic (no GPU) ------------------------------------------------------------- */
int64_t swec_expected_shard_size(int64_t dat_size, int data_shards, int64_t large_block,
                                 int64_t small_block);
typedef struct swec_interval {
    int32_t block_index;
    int32_t is_large_block;
    int64_t inner_block_offset;
    int64_t size;
    int32_t large_block_rows_count;
    int32_t reserved;
} swec_interval;
/* Returns the number of intervals written, or SWEC_ERR_INVALID_ARG if cap is too small.         */
int swec_locate_data(int64_t large_block, int64_t small_block, int64_t shard_dat_size,
                     int64_t offset, int64_t size, int data_shards, swec_interval *out, int cap);
void swec_interval_to_shard(const swec_interval *iv, int64_t large_block, int64_t small_block,
                            int data_shards, int *shard_id, int64_t *shard_offset);

/* ---- pinned host memory for callers that stage their own buffers ---------------------------- */
void *swec_alloc_pinned(size_t bytes);
/* Same, bound to the NUMA node the GPU `device` is attached to (full PCIe rate on 2-socket hosts). */
void *swec_alloc_pinned_for_device(int device, size_t bytes);
void swec_free_pinned(void *p);

/* ---- measurement helpers (synthetic volumes, device digests) -------------------------------- */
/* byte b of the stream = byte (b%8) of splitmix64(seed + (b/8 + 1)·0x9E3779B97F4A7C15).        */
int swec_synth_fill_device(int device, void *dst, uint64_t byte_offset, size_t bytes,
                           uint64_t seed, void *stream);
/* 64-bit order-sensitive digest of a device buffer; synchronises `stream`.                      */
int swec_digest_device(int device, const void *src, size_t bytes, uint64_t *digest, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SWEC_H */
