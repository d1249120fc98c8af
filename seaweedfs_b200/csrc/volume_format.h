// seaweedfs_b200/csrc/volume_format.h — the SeaweedFS volume format, stated once for the host code:
//   the two-tier striping of a .dat into k data shards       weed/storage/erasure_coding/ec_encoder.go:280-321
//   the default geometry and ratio                            ec_encoder.go:25-26, 61-69
//   the .ecNN shard files, findShardFile, the ratio in .vif   ec_encoder.go:76-108, 131-169
//   the 16-byte .idx / .ecx entries and the .ecj journal      weed/storage/types/needle_types.go, ec_volume.go:419-458
// Host-only: no CUDA here.  What a caller does with a row count, a path or an entry stays with the caller.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/swec.h"
#include "needle_format.h"  // the needle record itself, and GetActualSize

namespace swec {

// WriteEcFilesWithContext: 1 GiB / 1 MiB blocks, 256 KiB buffers, 10+4 (ec_encoder.go:25-26, 61-69)
constexpr int64_t kLargeBlockSize = int64_t(1) << 30;
constexpr int64_t kSmallBlockSize = int64_t(1) << 20;
constexpr int64_t kBufferSize = 256 * 1024;
constexpr int kDefaultDataShards = 10, kDefaultParityShards = 4;

// encodeDatFile's striping of a .dat of `dat_size` bytes: rows of k large blocks while a whole large row remains,
// then rows of k small blocks; the last small row may be partial (`tail` bytes), and shard i holds the bytes of
// block i of every row.  A shard is `shard_size()` bytes: the tail row counts as a whole small row.
struct StripeGeometry {
    int64_t large, small;
    int k;
    int64_t large_rows = 0;  // rows of k large blocks
    int64_t small_rows = 0;  // full rows of k small blocks
    int64_t tail = 0;        // bytes of the last, partial small row (0 = none)

    StripeGeometry(int64_t dat_size, int k_, int64_t large_, int64_t small_) : large(large_), small(small_), k(k_) {
        large_rows = dat_size / large_row();
        const int64_t rem = dat_size - large_rows * large_row();
        small_rows = rem / small_row();
        tail = rem - small_rows * small_row();
    }

    int64_t large_row() const { return large * k; }
    int64_t small_row() const { return small * k; }
    int64_t small_dat_offset() const { return large_rows * large_row(); }  // where the small rows start, in the .dat
    int64_t tail_dat_offset() const { return small_dat_offset() + small_rows * small_row(); }
    int64_t small_shard_offset() const { return large_rows * large; }  // ... and in every shard
    int64_t tail_shard_offset() const { return small_shard_offset() + small_rows * small; }
    int64_t shard_size() const { return tail_shard_offset() + (tail > 0 ? small : 0); }
    // bytes of the tail row that fall to shard i; the rest of its block is zero padding
    int64_t tail_bytes(int i) const { return std::clamp<int64_t>(tail - int64_t(i) * small, 0, small); }
};

// where a .dat byte range lies: LocateData + ToShardIdAndOffset (ec_locate.go:16-98) on the default block sizes cut the
// `size` bytes at `offset` into (shard, shard offset, length) pieces, in .dat order; the status is swec_locate_data's
struct Chunk { int shard; int64_t offset, size; };
int locate_chunks(int64_t shard_dat_size, int k, int64_t offset, int64_t size, std::vector<Chunk>* out);

// ---- shard files

std::string shard_ext(int i);              // ToExt: ".ec00" .. (ec_encoder.go:106-108)
bool is_file(const std::string& path);     // exists and is not a directory
// findShardFile (ec_encoder.go:131-169): <base>.ecNN, else <dir>/<basename(base)>.ecNN for each of the dirs in
// order; empty when there is none
std::string find_shard_file(const std::string& base, const char* const* dirs, int ndirs, int i);
int shard_size_error(int64_t expected, int64_t actual);  // SWEC_ERR_SHARD_SIZE, with the reference's text
// rebuildEcFiles (ec_encoder.go:323-377): every shard has the length of the first one checked (*size < 0: none yet)
int check_length(int fd, int64_t* size);
// the index base a handler works on: index_base when given, else data_base; with `fallback` also data_base when
// <index_base>.ecx does not exist (NewEcVolume, ec_volume.go:72-85; volume_grpc_erasure_coding.go:211-217,608-611)
std::string index_base_of(const char* data_base, const char* index_base, bool fallback);

// ---- .vif: protobuf-JSON of VolumeInfo (weed/storage/volume_info/volume_info.go:73-95)

// what NewEcVolume loads from .vif (ec_volume.go:114-154): the EC ratio from a valid <data_base>.vif, else 10+4; the
// needle version and datFileSize (0 = absent) from <data_base>.vif when it can be opened, else from <index_base>.vif
struct VolumeInfo { int k, m; int64_t version, dat_file_size; };
VolumeInfo read_volume_info(const std::string& data_base, const std::string& index_base);
// the EC ratio of a volume (volume_grpc_erasure_coding.go:61-77, ec_encoder.go:76-95)
void ec_ratio(const std::string& base, int* k, int* m);
// SaveVolumeInfo (volume_info.go:73-95), written in place
int save_volume_info(const std::string& path, uint32_t version, int64_t dat_size, uint64_t expire_at_sec, int ds, int ps);

// ---- index entries: 8-byte needle id, 4-byte offset in units of 8 bytes, 4-byte size, all big-endian
//      (needle_types.go:58-64, offset_4bytes.go:14-60, needle_map/needle_value.go:24-30)

constexpr int kIndexEntrySize = 16;   // NeedleMapEntrySize
constexpr int32_t kTombstone = -1;    // TombstoneFileSize

inline uint64_t be64(const uint8_t* p) {
    uint64_t v = 0;
    for (int i = 0; i < 8; i++) v = (v << 8) | p[i];
    return v;
}
inline uint32_t be32(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }
inline void put_be64(uint8_t* p, uint64_t v) {
    for (int i = 7; i >= 0; i--) { p[i] = uint8_t(v); v >>= 8; }
}
inline void put_be32(uint8_t* p, uint32_t v) {
    for (int i = 3; i >= 0; i--) { p[i] = uint8_t(v); v >>= 8; }
}
inline bool size_deleted(int32_t s) { return s < 0 || s == kTombstone; }  // Size.IsDeleted, needle_types.go:25-27

struct IndexEntry {
    uint64_t key;
    int64_t offset;  // in bytes: Offset.ToActualOffset
    int32_t size;
};
inline IndexEntry index_entry(const uint8_t* p) { return {be64(p), int64_t(be32(p + 8)) * 8, int32_t(be32(p + 12))}; }

// SearchNeedleFromSortedIndex (ec_volume.go:431-458): the entry number of `key` in a sorted index, or -1
int64_t search_sorted_index(const uint8_t* index, int64_t entries, uint64_t key);

// the needle ids of a .ecj deletion journal: 8 bytes each, big-endian; a trailing partial id is ignored
std::vector<uint64_t> ecj_ids(const std::vector<uint8_t>& ecj);

bool read_file(const std::string& path, std::vector<uint8_t>* out);  // the whole file; false when it cannot be opened
// the findings text of a check into the caller's errors[errors_cap]: cut at errors_cap - 1 bytes and NUL-terminated
void copy_findings(const std::string& text, char* errors, size_t errors_cap);

// FindDatFileSize (ec_decoder.go:113-135) with the needle version given: the end of the furthest live needle of
// <index_base>.ecx, at least the superblock
int dat_file_size_from_ecx(const std::string& index_base, int version, int64_t* dat_size);

}  // namespace swec
