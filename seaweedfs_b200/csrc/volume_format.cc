// seaweedfs_b200/csrc/volume_format.cc — see volume_format.h; also the layout arithmetic of the C ABI
// (swec_expected_shard_size, swec_locate_data, swec_interval_to_shard).
#include "volume_format.h"

#include <libgen.h>
#include <sys/stat.h>

#include <cerrno>
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

// .vif is protobuf-JSON (weed/storage/volume_info/volume_info.go:73-95); we only need
// ecShardConfig.{dataShards,parityShards} (weed/pb/volume_server.proto:561-577).
bool read_vif_ratio(const std::string& path, int* ds, int* ps) {
    std::vector<uint8_t> raw;
    if (!read_file(path, &raw)) return false;
    const std::string txt(raw.begin(), raw.end());
    int64_t a = 0, b = 0;
    if (!mini_json::nested_int(txt, "ecShardConfig", "ec_shard_config", "dataShards", "data_shards", &a) ||
        !mini_json::nested_int(txt, "ecShardConfig", "ec_shard_config", "parityShards", "parity_shards", &b))
        return false;
    if (a < 0 || b < 0 || a > 255 || b > 255) return false;
    *ds = int(a);
    *ps = int(b);
    return true;
}

void ec_ratio(const std::string& base, int* k, int* m) {
    int ds = 0, ps = 0;
    if (read_vif_ratio(base + ".vif", &ds, &ps) && ds > 0 && ps > 0 && ds + ps <= SWEC_MAX_SHARDS) {
        *k = ds;
        *m = ps;
    } else {
        *k = kDefaultDataShards;
        *m = kDefaultParityShards;
    }
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
