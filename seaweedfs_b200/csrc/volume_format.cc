// seaweedfs_b200/csrc/volume_format.cc — see volume_format.h; also the layout arithmetic of the C ABI
// (swec_expected_shard_size, swec_locate_data, swec_interval_to_shard).
#include "volume_format.h"

#include <fcntl.h>
#include <libgen.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cerrno>
#include <cinttypes>
#include <cstdio>
#include <cstring>

#include "engine.h"
#include "mini_json.h"

namespace swec {

std::string shard_ext(int i) {
    char b[16];
    snprintf(b, sizeof b, ".ec%02d", i);
    return b;
}

bool is_file(const std::string& path) {
    struct stat st;
    return stat(path.c_str(), &st) == 0 && !S_ISDIR(st.st_mode);
}

std::string find_shard_file(const std::string& base, const char* const* dirs, int ndirs, int i) {
    const std::string own = base + shard_ext(i);
    if (is_file(own)) return own;
    std::string base_copy(base);
    const std::string base_name = basename(&base_copy[0]);
    for (int d = 0; d < ndirs; d++) {
        const std::string cand = std::string(dirs[d]) + "/" + base_name + shard_ext(i);
        if (is_file(cand)) return cand;
    }
    return "";
}

int shard_size_error(int64_t expected, int64_t actual) {
    return fail(SWEC_ERR_SHARD_SIZE, "ec shard size expected " + std::to_string(expected) + " actual " + std::to_string(actual));
}

int check_length(int fd, int64_t* size) {
    struct stat st;
    if (fstat(fd, &st) != 0) return fail(SWEC_ERR_IO, std::string("fstat shard: ") + strerror(errno));
    if (*size < 0) *size = st.st_size;
    return *size == st.st_size ? SWEC_OK : shard_size_error(*size, st.st_size);
}

std::string index_base_of(const char* data_base, const char* index_base, bool fallback) {
    const std::string ib(index_base && *index_base ? index_base : data_base);
    return fallback && !is_file(ib + ".ecx") ? std::string(data_base) : ib;
}

void ec_ratio(const std::string& base, int* k, int* m) {
    const VolumeInfo vi = read_volume_info(base, base);
    *k = vi.k;
    *m = vi.m;
}

VolumeInfo read_volume_info(const std::string& data_base, const std::string& index_base) {
    std::vector<uint8_t> raw;
    const bool own = read_file(data_base + ".vif", &raw);
    std::string txt(raw.begin(), raw.end());
    // ecShardConfig (weed/pb/volume_server.proto:561-577), when it is a ratio the codec takes
    int64_t a = 0, b = 0, version = 0, dat_size = 0;
    const bool ratio = mini_json::nested_int(txt, "ecShardConfig", "ec_shard_config", "dataShards", "data_shards", &a) &&
                       mini_json::nested_int(txt, "ecShardConfig", "ec_shard_config", "parityShards", "parity_shards", &b) &&
                       a > 0 && b > 0 && a < SWEC_MAX_SHARDS && b <= SWEC_MAX_SHARDS - a;
    if (own || read_file(index_base + ".vif", &raw)) {  // 64-bit integers are rendered as strings
        txt.assign(raw.begin(), raw.end());
        mini_json::top_int(txt, "version", nullptr, &version);
        mini_json::top_int(txt, "datFileSize", "dat_file_size", &dat_size);
    }
    return {ratio ? int(a) : kDefaultDataShards, ratio ? int(b) : kDefaultParityShards, version, dat_size};
}

// protojson with EmitUnpopulated and a two-space indent.  protojson renders 64-bit integers as strings and deliberately
// does not promise byte-stable whitespace, so readers (ours: read_volume_info; Go: protojson.Unmarshal) parse, not
// compare.
int save_volume_info(const std::string& path, uint32_t version, int64_t dat_size, uint64_t expire_at_sec, int ds, int ps) {
    struct stat st;
    if (stat(path.c_str(), &st) == 0 && access(path.c_str(), W_OK) != 0)
        return fail(SWEC_ERR_IO, "failed to check " + path + " not writable");
    char text[512];
    const int n = snprintf(text, sizeof text,
                           "{\n"
                           "  \"files\": [],\n"
                           "  \"version\": %u,\n"
                           "  \"replication\": \"\",\n"
                           "  \"bytesOffset\": 0,\n"
                           "  \"datFileSize\": \"%" PRId64 "\",\n"
                           "  \"expireAtSec\": \"%" PRIu64 "\",\n"
                           "  \"readOnly\": false,\n"
                           "  \"ecShardConfig\": {\n"
                           "    \"dataShards\": %d,\n"
                           "    \"parityShards\": %d\n"
                           "  }\n"
                           "}",
                           version, dat_size, expire_at_sec, ds, ps);
    const int fd = open(path.c_str(), O_TRUNC | O_CREAT | O_WRONLY, 0644);
    if (fd < 0) return fail(SWEC_ERR_IO, "failed to write " + path + ": " + strerror(errno));
    int put = 0;
    while (put < n) {
        const ssize_t w = write(fd, text + put, size_t(n - put));
        if (w < 0) {
            if (errno == EINTR) continue;
            const int e = errno;
            close(fd);
            return fail(SWEC_ERR_IO, "failed to write " + path + ": " + strerror(e));
        }
        put += int(w);
    }
    close(fd);
    return SWEC_OK;
}

int64_t search_sorted_index(const uint8_t* index, int64_t entries, uint64_t key) {
    int64_t lo = 0, hi = entries;
    while (lo < hi) {
        const int64_t mid = (lo + hi) / 2;
        const uint64_t k = be64(index + mid * kIndexEntrySize);
        if (k == key) return mid;
        if (k < key) lo = mid + 1;
        else hi = mid;
    }
    return -1;
}

std::vector<uint64_t> ecj_ids(const std::vector<uint8_t>& ecj) {
    std::vector<uint64_t> ids;
    ids.reserve(ecj.size() / 8);
    for (size_t off = 0; off + 8 <= ecj.size(); off += 8) ids.push_back(be64(&ecj[off]));
    return ids;
}

bool read_file(const std::string& path, std::vector<uint8_t>* out) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    uint8_t buf[1 << 16];
    size_t n;
    out->clear();
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) out->insert(out->end(), buf, buf + n);
    fclose(f);
    return true;
}

void copy_findings(const std::string& text, char* errors, size_t errors_cap) {
    if (!errors || !errors_cap) return;
    const size_t m = std::min(text.size(), errors_cap - 1);
    memcpy(errors, text.data(), m);
    errors[m] = 0;
}

int locate_chunks(int64_t shard_dat_size, int k, int64_t offset, int64_t size, std::vector<Chunk>* out) {
    // a read of `size` bytes crosses at most size / small + 2 blocks
    std::vector<swec_interval> ivs(size_t((size > 0 ? size : 0) / kSmallBlockSize) + 4);
    const int n = swec_locate_data(kLargeBlockSize, kSmallBlockSize, shard_dat_size, offset, size, k, ivs.data(), int(ivs.size()));
    out->clear();
    if (n < 0) return n;
    for (int j = 0; j < n; j++) {
        Chunk c{0, 0, ivs[size_t(j)].size};
        swec_interval_to_shard(&ivs[size_t(j)], kLargeBlockSize, kSmallBlockSize, k, &c.shard, &c.offset);
        out->push_back(c);
    }
    return SWEC_OK;
}

}  // namespace swec

using namespace swec;

extern "C" {

int64_t swec_expected_shard_size(int64_t dat_size, int k, int64_t large, int64_t small) {
    if (k <= 0 || large <= 0 || small <= 0 || dat_size < 0) return 0;
    return StripeGeometry(dat_size, k, large, small).shard_size();
}

int swec_locate_data(int64_t large, int64_t small, int64_t shard_dat_size, int64_t offset, int64_t size, int k,
                     swec_interval* out, int cap) {
    if (large <= 0 || small <= 0 || k <= 0 || !out) return fail(SWEC_ERR_INVALID_ARG, "bad argument");
    const int64_t nlarge_rows = shard_dat_size / large;  // ec_locate.go:67
    const int64_t large_area = nlarge_rows * large * k;
    bool is_large = offset < large_area;
    const int64_t rel = is_large ? offset : offset - large_area;
    const int64_t blk = is_large ? large : small;
    int64_t block_index = rel / blk, inner = rel % blk;
    int n = 0;
    while (size > 0) {
        const int64_t room = (is_large ? large : small) - inner;
        if (room > 0) {
            if (n >= cap) return fail(SWEC_ERR_INVALID_ARG, "interval buffer too small");
            swec_interval& iv = out[n++];
            iv.block_index = int32_t(block_index);
            iv.is_large_block = is_large ? 1 : 0;
            iv.inner_block_offset = inner;
            iv.large_block_rows_count = int32_t(nlarge_rows);
            iv.reserved = 0;
            iv.size = std::min(size, room);
            size -= iv.size;
            if (size == 0) break;
        }
        // moveToNextBlock (ec_locate.go:55-63): the block after the last large one is small block 0
        block_index++;
        if (is_large && block_index == nlarge_rows * k) {
            is_large = false;
            block_index = 0;
        }
        inner = 0;
    }
    return n;
}

void swec_interval_to_shard(const swec_interval* iv, int64_t large, int64_t small, int k, int* shard_id,
                            int64_t* shard_offset) {
    const int64_t row = iv->block_index / k;  // ec_locate.go:87-98
    int64_t off = iv->inner_block_offset;
    off += iv->is_large_block ? row * large : int64_t(iv->large_block_rows_count) * large + row * small;
    if (shard_id) *shard_id = iv->block_index % k;
    if (shard_offset) *shard_offset = off;
}

}  // extern "C"
