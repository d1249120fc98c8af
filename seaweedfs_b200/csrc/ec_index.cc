// seaweedfs_b200/csrc/ec_index.cc — the index files either side of the RS path (SURVEY §8f row 4,
// Appendix C).  No GF arithmetic here: host-only twins of
//   WriteSortedFileFromIdx / readNeedleMap        weed/storage/erasure_coding/ec_encoder.go:31-58,379-396
//   RebuildEcxFile / MarkNeedleDeleted            weed/storage/erasure_coding/ec_volume_delete.go:13-26,95-142
//   SearchNeedleFromSortedIndex                   weed/storage/erasure_coding/ec_volume.go:431-458
//   WriteIdxFileFromEcIndex, FindDatFileSize, HasLiveNeedles   weed/storage/erasure_coding/ec_decoder.go:23-92
// so that a volume server using libswec for ec.encode / ec.rebuild / ec.decode needs nothing else
// from the Go package for these files.  Entry format (4-byte offsets, the default build):
// 8-byte needle id, 4-byte offset in units of 8 bytes, 4-byte size, all big-endian
// (weed/storage/types/needle_types.go:58-64, offset_4bytes.go:14-60, needle_map/needle_value.go:24-30).
#include <errno.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "engine.h"
#include "volume_format.h"

namespace swec {
namespace {

constexpr int64_t kSuperBlockSize = 8; // super_block.SuperBlockSize

// Replaces `path` atomically: the bytes go to <path>.tmp.<pid>, which is renamed over the target.  A mounted
// EcVolume maps .ecx MAP_SHARED (ec_volume.cc) and binary-searches the mapping; rewriting the same inode in place
// (O_TRUNC) while it is mounted — ec.encode re-run on a mounted volume — would leave the search touching pages past
// the new EOF: SIGBUS, which kills the whole volume server where the reference's ReadAt only returns an error.
// With rename() existing mappings keep the old inode and its bytes until they are unmapped.
bool write_all(const std::string& path, const std::vector<uint8_t>& data) {
    static std::atomic<unsigned> serial{0};  // two threads of one process may rewrite the same path
    const std::string tmp = path + ".tmp." + std::to_string(long(getpid())) + "." + std::to_string(serial++);
    const int fd = open(tmp.c_str(), O_TRUNC | O_CREAT | O_WRONLY, 0644);
    if (fd < 0) return false;
    size_t put = 0;
    while (put < data.size()) {
        const ssize_t n = write(fd, data.data() + put, data.size() - put);
        if (n < 0) {
            if (errno == EINTR) continue;
            const int keep = errno;
            close(fd);
            unlink(tmp.c_str());
            errno = keep;
            return false;
        }
        put += size_t(n);
    }
    if (close(fd) != 0 || rename(tmp.c_str(), path.c_str()) != 0) {
        const int keep = errno;
        unlink(tmp.c_str());
        errno = keep;
        return false;
    }
    return true;
}

bool exists(const std::string& p) {
    struct stat st;
    return stat(p.c_str(), &st) == 0;
}

int io_err(const std::string& what) { return fail(SWEC_ERR_IO, what + ": " + strerror(errno)); }

}  // namespace
}  // namespace swec

using namespace swec;

extern "C" {

int swec_write_sorted_file_from_idx(const char* base, const char* ext) {
    if (!base || !ext) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    std::vector<uint8_t> idx;
    if (!read_file(std::string(base) + ".idx", &idx)) return io_err(std::string("cannot read Volume Index ") + base + ".idx");
    // readNeedleMap replays the .idx into a map: a live entry (non-zero offset, size not deleted) sets the key, anything
    // else removes it — so the LAST entry of a key alone decides whether and how the key appears.  Sorting the entries
    // by (key, position) and keeping each key's last one gives the same file without a 30-million-node tree for a
    // full 30 GB volume of small needles.
    struct E { uint64_t key; uint32_t pos, offset, size; };
    const size_t n = idx.size() / kIndexEntrySize;
    if (n > 0xFFFFFFFFull) return fail(SWEC_ERR_INVALID_ARG, "index too large");
    std::vector<E> es(n);
    for (size_t i = 0; i < n; i++) {
        const uint8_t* p = &idx[i * kIndexEntrySize];
        es[i] = {be64(p), uint32_t(i), be32(p + 8), be32(p + 12)};
    }
    std::sort(es.begin(), es.end(), [](const E& a, const E& b) { return a.key != b.key ? a.key < b.key : a.pos < b.pos; });
    std::vector<uint8_t> out;
    out.reserve(n * kIndexEntrySize);
    for (size_t i = 0; i < n; i++) {
        if (i + 1 < n && es[i + 1].key == es[i].key) continue;  // not the key's last word
        const E& e = es[i];
        if (e.offset == 0 || size_deleted(int32_t(e.size))) continue;  // the key ends deleted
        uint8_t rec[kIndexEntrySize];
        put_be64(rec, e.key);
        put_be32(rec + 8, e.offset);
        put_be32(rec + 12, e.size);
        out.insert(out.end(), rec, rec + kIndexEntrySize);  // ascending keys: AscendingVisit
    }
    if (!write_all(std::string(base) + ext, out)) return io_err("failed to open ecx file");
    return SWEC_OK;
}

int swec_rebuild_ecx_file(const char* base) {
    if (!base) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    const std::string b(base);
    if (!exists(b + ".ecj")) return SWEC_OK;
    const int ecx = open((b + ".ecx").c_str(), O_RDWR);
    if (ecx < 0) return io_err("rebuild: failed to open ecx file");
    std::vector<uint8_t> index, ecj;
    if (!read_file(b + ".ecx", &index)) {
        close(ecx);
        return io_err("rebuild: failed to read ecx file");
    }
    const int64_t entries = int64_t(index.size()) / kIndexEntrySize;
    if (!read_file(b + ".ecj", &ecj)) {
        close(ecx);
        return io_err("rebuild: failed to open ecj file");
    }
    // SearchNeedleFromSortedIndex + MarkNeedleDeleted for every journalled id: the search runs on the copy in
    // memory (a 30 GB volume of small needles has a 480 MB index and 25 probes per id), the tombstone is written
    // in place on disk, exactly the four size bytes the reference rewrites
    for (const uint64_t id : ecj_ids(ecj)) {
        const int64_t at = search_sorted_index(index.data(), entries, id);
        if (at < 0) continue;
        uint8_t t[4];
        put_be32(t, uint32_t(kTombstone));
        if (memcmp(&index[size_t(at) * kIndexEntrySize + 12], t, 4) != 0) {
            memcpy(&index[size_t(at) * kIndexEntrySize + 12], t, 4);
            if (pwrite(ecx, t, 4, off_t(at * kIndexEntrySize + 12)) != 4) {
                close(ecx);
                return io_err("sorted needle write error");
            }
        }
    }
    close(ecx);
    unlink((b + ".ecj").c_str());
    return SWEC_OK;
}

int swec_write_idx_file_from_ec_index(const char* base) {
    if (!base) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    const std::string b(base);
    std::vector<uint8_t> data;
    if (!read_file(b + ".ecx", &data)) return io_err("cannot open ec index " + b + ".ecx");
    std::vector<uint8_t> ecj;
    if (exists(b + ".ecj") && !read_file(b + ".ecj", &ecj)) return io_err("cannot open ec index " + b + ".ecj");
    for (const uint64_t id : ecj_ids(ecj)) {  // one tombstone entry per journalled id
        uint8_t e[kIndexEntrySize] = {0};
        put_be64(e, id);
        put_be32(e + 12, uint32_t(kTombstone));
        data.insert(data.end(), e, e + kIndexEntrySize);
    }
    if (!write_all(b + ".idx", data)) return io_err("cannot open " + b + ".idx");
    return SWEC_OK;
}

int swec_has_live_needles(const char* index_base, int* has_live) {
    if (!index_base || !has_live) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    std::vector<uint8_t> ecx;
    if (!read_file(std::string(index_base) + ".ecx", &ecx)) return io_err(std::string("cannot open ec index ") + index_base + ".ecx");
    *has_live = 0;
    for (size_t off = 0; off + kIndexEntrySize <= ecx.size(); off += kIndexEntrySize)
        if (!size_deleted(index_entry(&ecx[off]).size)) {
            *has_live = 1;
            break;
        }
    return SWEC_OK;
}

// idx.CheckIndexFile (weed/storage/idx/check.go:36-111) — what EcVolume.ScrubIndex runs on .ecx
// (ec_volume_scrub.go:20-25): entries sorted by (offset, size); two neighbours overlap when the later one starts at
// or before the end of the earlier one; and the file must be a whole number of entries.
int swec_check_index_file(const char* path, int needle_version, int64_t* entries, char* errors, size_t errors_cap,
                          int* n_errors) {
    if (!path || !entries || !n_errors) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    std::vector<uint8_t> raw;
    if (!read_file(path, &raw)) return io_err(std::string("cannot read index ") + path);
    struct E { int index; uint64_t id; int64_t offset; int32_t size; };
    std::vector<E> es;
    for (size_t off = 0; off + kIndexEntrySize <= raw.size(); off += kIndexEntrySize) {  // WalkIndexFile ignores a trailing partial entry
        const IndexEntry x = index_entry(&raw[off]);
        es.push_back({int(es.size()), x.key, x.offset, x.size});
    }
    std::stable_sort(es.begin(), es.end(), [](const E& a, const E& b) { return a.offset != b.offset ? a.offset < b.offset : a.size < b.size; });
    // needle.GetActualSize with the reference's types: PaddingLength is computed in Size (int32) arithmetic and wraps
    // like Go does; NeedleBodyLength adds in int64 (needle_read_tail.go:36-49)
    auto actual = [&](int32_t size) -> int64_t {
        const uint32_t tail = needle_version == 3 ? 4u + 8u : 4u;
        const int32_t sum = int32_t(16u + uint32_t(size) + tail);  // wraps
        const int32_t padding = 8 - (sum % 8);                      // Go's % keeps the sign of the dividend, like C++
        return 16 + int64_t(size) + int64_t(tail) + int64_t(padding);
    };
    std::string text;
    int count = 0;
    auto add = [&](const std::string& m) {
        if (count++) text += "\n";
        text += m;
    };
    for (size_t i = 1; i < es.size(); i++) {
        const E &e = es[i], &last = es[i - 1];
        int64_t end = e.offset, last_end = last.offset;
        if (const int64_t sz = actual(e.size)) end += sz - 1;
        if (const int64_t sz = actual(last.size)) last_end += sz - 1;
        if (e.offset <= last_end)
            add("needle " + std::to_string(e.id) + " (#" + std::to_string(e.index + 1) + ") at [" + std::to_string(e.offset) + "-" +
                std::to_string(end) + "] overlaps needle " + std::to_string(last.id) + " at [" + std::to_string(last.offset) + "-" +
                std::to_string(last_end) + "]");
    }
    const int64_t n = int64_t(es.size());
    if (n * kIndexEntrySize != int64_t(raw.size()))
        add("expected an index file of size " + std::to_string(raw.size()) + ", got " + std::to_string(n * kIndexEntrySize));
    *entries = n;
    *n_errors = count;
    copy_findings(text, errors, errors_cap);
    return SWEC_OK;
}

int swec_find_dat_file_size(const char* data_base, const char* index_base, int64_t* dat_size) {
    if (!data_base || !index_base || !dat_size) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    // readEcVolumeVersion: the superblock sits at the start of .ec00; byte 0 is the needle version
    const int fd = open((std::string(data_base) + ".ec00").c_str(), O_RDONLY);
    if (fd < 0) return io_err(std::string("open ec volume ") + data_base + " superblock");
    uint8_t sb[kSuperBlockSize];
    const ssize_t got = pread(fd, sb, sizeof sb, 0);
    close(fd);
    if (got != ssize_t(sizeof sb)) return fail(SWEC_ERR_IO, "cannot read the superblock from .ec00");
    return swec::dat_file_size_from_ecx(index_base, sb[0], dat_size);
}

}  // extern "C"

namespace swec {

int dat_file_size_from_ecx(const std::string& index_base, int version, int64_t* dat_size) {
    std::vector<uint8_t> ecx;
    if (!read_file(index_base + ".ecx", &ecx)) return io_err("cannot open ec index " + index_base + ".ecx");
    int64_t size = kSuperBlockSize;
    for (size_t off = 0; off + kIndexEntrySize <= ecx.size(); off += kIndexEntrySize) {
        const IndexEntry e = index_entry(&ecx[off]);
        if (size_deleted(e.size)) continue;
        const int64_t stop = e.offset + needle_actual_size(e.size, version);
        if (stop > size) size = stop;
    }
    *dat_size = size;
    return SWEC_OK;
}

}  // namespace swec
