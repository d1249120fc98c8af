// seaweedfs_b200/csrc/ec_volume.cc — the volume-server-local bodies of the three gRPC handlers that
// drive the RS path (SURVEY §8f row 1), as single C-ABI calls:
//   swec_ec_shards_generate    VolumeEcShardsGenerate   weed/server/volume_grpc_erasure_coding.go:43-146
//   swec_ec_shards_rebuild     VolumeEcShardsRebuild    weed/server/volume_grpc_erasure_coding.go:149-225
//   swec_ec_shards_heal        the same, rebuilding through swec_heal_ec_files: the damaged present shards corrected too
//   swec_ec_shards_to_volume   VolumeEcShardsToVolume   weed/server/volume_grpc_erasure_coding.go:578-668
//   swec_ec_shards_to_volume_checked   the same from any k shards, damaged data shards corrected on the GPU first
//   swec_read_ec_needles       Store.ReadEcShardNeedle + readEcShardIntervals + readOneEcShardInterval +
//                              recoverOneRemoteEcShardInterval, on local shard files, batched
//                                                       weed/storage/store_ec.go:252-355,482-560
// Everything the handlers do to FILES is here, in the reference's order (.ecx before the shards, the
// .dat size snapshot before encoding, .vif last, partial outputs removed on any error); what they do
// to the server's in-memory state (volume lookup, maintenance mode, disk-location scan, compaction)
// stays in Go.  The shard arithmetic runs on the GPU through swec_generate_ec_files /
// swec_rebuild_ec_files; the index and .vif work is host-only.
#include <errno.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <cinttypes>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "damage.h"
#include "engine.h"
#include "needle_damage.h"
#include "needles.h"
#include "sketch.h"
#include "volume_format.h"

namespace swec {

namespace {

// VolumeEcShardsToVolume's index steps (volume_grpc_erasure_coding.go:621-644): fold .ecj first so deleted needles are
// not counted live, refuse a volume without live needles, then FindDatFileSize (ec_decoder.go:94-135) with the needle
// version from the superblock of the shard file `ec00`, or from `version` when there is none
int decoded_dat_size(const std::string& ib, const std::string& ec00, int version, int64_t* size) {
    int rc = swec_rebuild_ecx_file(ib.c_str());
    if (rc) return rc;
    int live = 0;
    if ((rc = swec_has_live_needles(ib.c_str(), &live))) return rc;
    if (!live) return fail(SWEC_ERR_NO_LIVE_NEEDLES, "ec volume has no live entries");  // EcNoLiveEntriesSubstring
    if (ec00.empty()) return dat_file_size_from_ecx(ib, version, size);
    return swec_find_dat_file_size(ec00.substr(0, ec00.size() - 5).c_str(), ib.c_str(), size);
}

}  // namespace
}  // namespace swec

using namespace swec;

extern "C" {

int swec_ec_shards_generate(const char* data_base, const char* index_base, uint32_t needle_version,
                            uint64_t expire_at_sec, int device) {
    if (!data_base) return fail(SWEC_ERR_INVALID_ARG, "data_base_file_name is NULL");
    const std::string db(data_base), ib = index_base_of(data_base, index_base, false);
    int k, m;
    ec_ratio(db, &k, &m);

    struct Cleanup {  // the handler's deferred cleanup: shards and .ecx go away unless we reach the end
        const std::string &db, &ib;
        int total;
        bool armed = true;
        ~Cleanup() {
            if (!armed) return;
            const std::string keep = last_error();  // unlink() must not disturb the reported detail
            for (int i = 0; i < total; i++) unlink((db + shard_ext(i)).c_str());
            unlink((ib + ".ecx").c_str());
            set_last_error(keep);
        }
    } cleanup{db, ib, k + m};

    // .ecx BEFORE the shards (the race the reference documents at :82-95)
    int rc = swec_write_sorted_file_from_idx(ib.c_str(), ".ecx");
    if (rc) return rc;
    // snapshot of the .dat size before encoding — what .ecx references (:103)
    struct stat st;
    if (stat((db + ".dat").c_str(), &st) != 0) return fail(SWEC_ERR_IO, "failed to stat dat file " + db + ".dat: " + strerror(errno));
    if (needle_version == 0) {  // v.Version(): byte 0 of the superblock (super_block.go; ec_decoder.go:94-111)
        const int fd = open((db + ".dat").c_str(), O_RDONLY);
        uint8_t b0 = 0;
        if (fd < 0 || pread(fd, &b0, 1, 0) != 1) {
            const int e = errno;
            if (fd >= 0) close(fd);
            return fail(SWEC_ERR_IO, "cannot read the superblock of " + db + ".dat: " + strerror(e));
        }
        close(fd);
        needle_version = b0;
    }
    rc = swec_generate_ec_files(db.c_str(), kBufferSize, kLargeBlockSize, kSmallBlockSize, k, m, device);
    if (rc) return rc;
    rc = save_volume_info(db + ".vif", needle_version, int64_t(st.st_size), expire_at_sec, k, m);
    if (rc) return rc;
    cleanup.armed = false;
    return SWEC_OK;
}

int swec_ec_shards_rebuild(const char* data_base, const char* index_base, const char* const* additional_dirs,
                           int n_additional_dirs, int device, uint32_t* rebuilt, int* n_rebuilt) {
    if (!data_base || !rebuilt || !n_rebuilt) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    // RebuildEcFiles: ratio from data_base.vif or 10+4; inputs searched in data_base's directory, then
    // additional_dirs; outputs created next to data_base (:203-209)
    int rc = swec_rebuild_ec_files(data_base, additional_dirs, n_additional_dirs, 0, 0, device, rebuilt, n_rebuilt);
    if (rc) return rc;
    // RebuildEcxFile on the index base, falling back to the data directory (:211-217)
    return swec_rebuild_ecx_file(index_base_of(data_base, index_base, true).c_str());
}

int swec_ec_shards_heal(const char* data_base, const char* index_base, const char* const* additional_dirs,
                        int n_additional_dirs, int device, int radius, uint32_t* rebuilt, int* n_rebuilt,
                        swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges, int* ok) {
    if (!data_base || !rebuilt || !n_rebuilt) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    int rc = swec_heal_ec_files(data_base, additional_dirs, n_additional_dirs, 0, 0, device, radius, rebuilt, n_rebuilt,
                                report, ranges, ranges_cap, n_ranges, ok);
    if (rc) return rc;
    return swec_rebuild_ecx_file(index_base_of(data_base, index_base, true).c_str());
}

int swec_ec_shards_to_volume(const char* data_base, const char* index_base, const char* const* additional_dirs,
                             int n_additional_dirs, int64_t* dat_file_size) {
    if (!data_base || (n_additional_dirs > 0 && !additional_dirs)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    const std::string db(data_base);
    int k, m;
    ec_ratio(db, &k, &m);  // NewEcVolume loads the ratio from .vif (ec_volume.go:114-154)
    // CollectEcShards: every data shard must be found locally (:601-606)
    std::vector<std::string> names;
    for (int i = 0; i < k; i++) {
        const std::string path = find_shard_file(db, additional_dirs, n_additional_dirs, i);
        if (path.empty()) return fail(SWEC_ERR_TOO_FEW_SHARDS, "ec volume missing shard " + std::to_string(i));
        names.push_back(path);
    }
    const std::string ib = index_base_of(data_base, index_base, true);  // :608-611
    int64_t size = 0;
    int rc = decoded_dat_size(ib, names[0], 0, &size);
    if (rc) return rc;
    std::vector<const char*> cnames;
    for (const auto& s : names) cnames.push_back(s.c_str());
    if ((rc = swec_write_dat_file(db.c_str(), size, cnames.data(), k, kLargeBlockSize, kSmallBlockSize))) return rc;
    if ((rc = swec_write_idx_file_from_ec_index(ib.c_str()))) return rc;
    if (dat_file_size) *dat_file_size = size;
    return SWEC_OK;
}

// swec_ec_shards_to_volume from any k of the k+m shards, through swec_write_dat_file_checked: the data shards are
// corrected (or rebuilt) on the GPU before the .dat is written, and a volume left with uncorrectable columns gets
// neither .dat nor .idx, so the caller keeps its EC shards.
int swec_ec_shards_to_volume_checked(const char* data_base, const char* index_base, const char* const* additional_dirs,
                                     int n_additional_dirs, int device, int radius, int64_t* dat_file_size,
                                     swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges,
                                     int* ok) {
    if (!data_base || !ok || (n_additional_dirs > 0 && !additional_dirs)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    *ok = 0;
    int rc;
    if ((rc = DamageOut{report, ranges, ranges_cap, n_ranges}.check()) || (rc = check_radius(radius, 0))) return rc;
    const std::string db(data_base);
    int k, m;
    ec_ratio(db, &k, &m);
    std::vector<std::string> names(size_t(k + m));
    int found = 0;
    for (int i = 0; i < k + m; i++) {
        names[size_t(i)] = find_shard_file(db, additional_dirs, n_additional_dirs, i);
        found += names[size_t(i)].empty() ? 0 : 1;
    }
    if (found < k)
        return fail(SWEC_ERR_TOO_FEW_SHARDS, "ec volume " + db + " has " + std::to_string(found) + " of its " +
                                                 std::to_string(k + m) + " shards, needs at least " + std::to_string(k));
    const std::string ib = index_base_of(data_base, index_base, true);
    // FindDatFileSize reads the needle version from .ec00's superblock; without .ec00, .vif keeps it.  Known before
    // anything is written.
    int64_t version = 0;
    if (names[0].empty() && (version = read_volume_info(db, ib).version) <= 0)
        return fail(SWEC_ERR_TOO_FEW_SHARDS, "ec volume " + db + " has no .ec00 and no needle version in its .vif");
    int64_t size = 0;
    if ((rc = decoded_dat_size(ib, names[0], int(version), &size))) return rc;
    std::vector<const char*> cnames;
    for (const auto& s : names) cnames.push_back(s.empty() ? nullptr : s.c_str());
    if ((rc = swec_write_dat_file_checked(db.c_str(), size, cnames.data(), k, m, kLargeBlockSize, kSmallBlockSize, device,
                                          radius, report, ranges, ranges_cap, n_ranges, ok)))
        return rc;
    if ((rc = swec_write_idx_file_from_ec_index(ib.c_str()))) {
        *ok = 0;
        unlink((db + ".dat").c_str());
        unlink((ib + ".idx").c_str());
        return rc;
    }
    if (dat_file_size) *dat_file_size = size;
    return SWEC_OK;
}

// ---- EcVolume: the mounted state the read path works from (ec_volume.go:36-160) ------------------

}  // extern "C"

struct swec_ec_volume {
    std::mutex mu;
    int k = swec::kDefaultDataShards, m = swec::kDefaultParityShards, version = 3, device = 0;
    int64_t shard_dat_size = 0;
    std::string index_base;
    std::vector<int> shard_fd;  // total entries, -1 = not local
    // the sealed index is mapped, not copied: a full volume of small needles has a ~500 MB .ecx and a server mounts
    // hundreds of EC volumes; a lookup touches ~25 pages of the page cache (the reference does 25 ReadAt calls)
    const uint8_t* ecx_map = nullptr;
    size_t ecx_bytes = 0;
    std::vector<uint64_t> deleted;  // ids of .ecj, sorted and unique: the reference's in-memory deletedNeedles set
    struct JournalStamp {           // .ecj as deleted last saw it; size -1 = read it again
        int64_t size = -1, mtime_ns = 0;
        uint64_t inode = 0;
    } ecj_seen;
    swec_encoder* enc = nullptr;  // created on the first recovery, keeps its staging ring and kernels

    int64_t entries() const { return int64_t(ecx_bytes) / swec::kIndexEntrySize; }
    swec::IndexEntry entry(int64_t i) const { return swec::index_entry(ecx_map + i * swec::kIndexEntrySize); }
    int64_t find(uint64_t id) const { return swec::search_sorted_index(ecx_map, entries(), id); }  // entry number or -1
    bool journalled(uint64_t id) const { return std::binary_search(deleted.begin(), deleted.end(), id); }
    static JournalStamp stamp(const struct stat* st) {  // nullptr: there is no journal
        if (!st) return {0, 0, 0};
        return {int64_t(st->st_size), int64_t(st->st_mtim.tv_sec) * 1000000000ll + st->st_mtim.tv_nsec, uint64_t(st->st_ino)};
    }
    void refresh_journal();
    ~swec_ec_volume() {
        if (ecx_map && ecx_bytes) munmap(const_cast<uint8_t*>(ecx_map), ecx_bytes);
        for (int fd : shard_fd)
            if (fd >= 0) close(fd);
        if (enc) swec_encoder_free(enc);
    }
};

void swec_ec_volume::refresh_journal() {
    // the deletion journal grows while the volume is mounted (DeleteNeedleFromEcx appends to .ecj): pick up new
    // entries when the file moved — size, mtime or inode, so a journal folded and re-created to the same length is
    // seen too — the reference keeps the same set in memory (ec_volume.go:351-384)
    struct stat st;
    const JournalStamp now = stamp(stat((index_base + ".ecj").c_str(), &st) == 0 ? &st : nullptr);
    if (now.size == ecj_seen.size && now.mtime_ns == ecj_seen.mtime_ns && now.inode == ecj_seen.inode) return;
    std::vector<uint8_t> ecj;  // stays empty when the journal cannot be read
    if (now.size > 0) swec::read_file(index_base + ".ecj", &ecj);
    ecj_seen = now;
    deleted = swec::ecj_ids(ecj);
    std::sort(deleted.begin(), deleted.end());
    deleted.erase(std::unique(deleted.begin(), deleted.end()), deleted.end());
}

extern "C" {

int swec_ec_volume_open(const char* data_base, const char* index_base, const char* const* additional_dirs,
                        int n_additional_dirs, int device, swec_ec_volume** out) {
    if (!out) return fail(SWEC_ERR_INVALID_ARG, "out is NULL");
    *out = nullptr;
    if (!data_base || (n_additional_dirs > 0 && !additional_dirs)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    const std::string db(data_base), ib = index_base_of(data_base, index_base, true);
    std::unique_ptr<swec_ec_volume> v(new (std::nothrow) swec_ec_volume());
    if (!v) return fail(SWEC_ERR_NOMEM, "out of memory");
    v->device = device;
    v->index_base = ib;

    // what NewEcVolume loads: ratio, needle version and datFileSize from .vif (ec_volume.go:114-154)
    const VolumeInfo vif = read_volume_info(db, ib);
    v->k = vif.k;
    v->m = vif.m;
    if (vif.version > 0) v->version = int(vif.version);
    const int total = v->k + v->m;
    // local shards: data_base's directory, then the other disks
    v->shard_fd.assign(size_t(total), -1);
    int64_t ecd_file_size = -1;
    int nlocal = 0;
    for (int i = 0; i < total; i++) {
        const std::string path = find_shard_file(db, additional_dirs, n_additional_dirs, i);
        if (path.empty()) continue;
        const int fd = open(path.c_str(), O_RDONLY);
        if (fd < 0) continue;  // unreadable = not local; its intervals are recovered from the others
        v->shard_fd[size_t(i)] = fd;
        nlocal++;
        if (ecd_file_size < 0) {
            struct stat st;
            if (fstat(fd, &st) == 0) ecd_file_size = st.st_size;
        }
    }
    if (nlocal == 0) return fail(SWEC_ERR_TOO_FEW_SHARDS, "ec shard " + db + " not found");
    // LocateEcShardNeedleInterval: .vif's datFileSize is authoritative; old volumes fall back to the
    // shard file size minus one (ec_volume.go:399-417)
    v->shard_dat_size = vif.dat_file_size > 0 ? vif.dat_file_size / v->k : ecd_file_size - 1;
    {
        const int efd = open((ib + ".ecx").c_str(), O_RDONLY);
        if (efd < 0) return fail(SWEC_ERR_IO, "cannot open ec volume index " + ib + ".ecx: " + strerror(errno));
        struct stat st;
        if (fstat(efd, &st) != 0) {
            const int e = errno;
            close(efd);
            return fail(SWEC_ERR_IO, "can not stat ec volume index " + ib + ".ecx: " + strerror(e));
        }
        v->ecx_bytes = size_t(st.st_size);
        if (v->ecx_bytes) {  // MAP_SHARED: tombstones that RebuildEcxFile writes in place are seen
            void* m = mmap(nullptr, v->ecx_bytes, PROT_READ, MAP_SHARED, efd, 0);
            if (m == MAP_FAILED) {
                const int e = errno;
                close(efd);
                v->ecx_bytes = 0;
                return fail(SWEC_ERR_IO, "cannot map ec volume index " + ib + ".ecx: " + strerror(e));
            }
            v->ecx_map = static_cast<const uint8_t*>(m);
        }
        close(efd);
    }
    *out = v.release();
    return SWEC_OK;
}

void swec_ec_volume_close(swec_ec_volume* v) { delete v; }

int swec_ec_volume_read_needles(swec_ec_volume* v, swec_needle_read* reads, int n_reads) {
    if (!v || (n_reads > 0 && !reads)) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    std::lock_guard<std::mutex> lock(v->mu);
    const int k = v->k, total = v->k + v->m, version = v->version;
    v->refresh_journal();

    // ---- pass 1: locate every needle, read what is local, collect what must be recovered
    struct Recover {
        int read_idx;
        size_t buf_off, len;
        int shard;
        std::vector<std::vector<uint8_t>> bufs;  // total entries; empty = not available
        std::vector<uint8_t*> ptrs;
        std::vector<uint8_t> present;
    };
    std::vector<Recover> recs;
    std::vector<Chunk> chunks;
    for (int r = 0; r < n_reads; r++) {
        swec_needle_read& rd = reads[r];
        rd.offset = 0;
        rd.size = 0;
        rd.n_bytes = 0;
        rd.n_recovered_intervals = 0;
        rd.status = SWEC_OK;
        const int64_t found = v->find(rd.needle_id);
        if (found < 0) {
            rd.status = SWEC_ERR_NOT_FOUND;
            continue;
        }
        const IndexEntry entry = v->entry(found);
        const int64_t offset = entry.offset;
        int32_t size = entry.size;
        if (v->journalled(rd.needle_id)) size = kTombstone;  // FindNeedleFromEcx (ec_volume.go:419-429)
        rd.offset = offset;
        rd.size = size;
        if (size_deleted(size)) {
            rd.status = SWEC_ERR_DELETED;
            continue;
        }
        // LocateEcShardNeedle passes GetActualSize(size) to LocateEcShardNeedleInterval, which applies
        // GetActualSize AGAIN (ec_volume.go:395,414): the reference reads a little past the record.  Kept,
        // because ReadEcShardNeedle returns len(bytes) and n.ReadBytes only parses the front.
        const int64_t want = needle_actual_size(needle_actual_size(size, version), version);
        if (!rd.buf || size_t(want) > rd.capacity) {
            rd.n_bytes = size_t(want);
            rd.status = SWEC_ERR_INVALID_ARG;
            continue;
        }
        if (const int rc = locate_chunks(v->shard_dat_size, k, offset, want, &chunks)) {
            rd.status = rc;
            continue;
        }
        size_t pos = 0;
        for (const auto& [sid, soff, bytes] : chunks) {
            const size_t len = size_t(bytes);
            bool ok = false;
            if (v->shard_fd[size_t(sid)] >= 0) {  // readLocalEcShardInterval (store_ec.go:407-422): all or nothing
                const ssize_t got = pread(v->shard_fd[size_t(sid)], rd.buf + pos, len, off_t(soff));
                ok = got == ssize_t(len);
            }
            if (!ok) {  // recoverOneRemoteEcShardInterval, with "remote" = every other local shard file
                Recover rc;
                rc.read_idx = r;
                rc.buf_off = pos;
                rc.len = len;
                rc.shard = sid;
                rc.bufs.resize(size_t(total));
                rc.present.assign(size_t(total), 0);
                int have = 0;
                for (int i = 0; i < total; i++) {
                    if (i == sid || v->shard_fd[size_t(i)] < 0) continue;
                    rc.bufs[size_t(i)].resize(len);
                    if (pread(v->shard_fd[size_t(i)], rc.bufs[size_t(i)].data(), len, off_t(soff)) == ssize_t(len)) {
                        rc.present[size_t(i)] = 1;
                        have++;
                    } else {
                        rc.bufs[size_t(i)].clear();  // nRead != len(buf): not available
                    }
                }
                if (have < k) {
                    rd.status = SWEC_ERR_TOO_FEW_SHARDS;
                    set_last_error("cannot recover shard " + std::to_string(sid) + ": only " + std::to_string(have) +
                                   " shards available, need at least " + std::to_string(k));
                    break;
                }
                for (int i = 0; i < k; i++)  // ReconstructData fills every missing DATA shard
                    if (!rc.present[size_t(i)]) rc.bufs[size_t(i)].resize(len);
                recs.push_back(std::move(rc));
                rd.n_recovered_intervals++;
            }
            pos += len;
        }
        if (rd.status == SWEC_OK) rd.n_bytes = pos;
    }

    // ---- pass 2: every interval that needs the arithmetic, in ONE batched ReconstructData on the GPU
    if (!recs.empty()) {
        if (!v->enc) {
            const int rc = swec_encoder_new(v->k, v->m, v->device, &v->enc);
            if (rc) return rc;
        }
        std::vector<swec_reconstruct_item> items(recs.size());
        for (size_t j = 0; j < recs.size(); j++) {
            recs[j].ptrs.assign(size_t(total), nullptr);
            for (int i = 0; i < total; i++)
                if (!recs[j].bufs[size_t(i)].empty()) recs[j].ptrs[size_t(i)] = recs[j].bufs[size_t(i)].data();
            items[j].shards = recs[j].ptrs.data();
            items[j].present = recs[j].present.data();
            items[j].shard_len = recs[j].len;
            items[j].data_only = 1;
        }
        const int rc = swec_reconstruct_batch(v->enc, items.data(), int(items.size()));
        if (rc) return rc;
        for (const Recover& rcv : recs) {
            swec_needle_read& rd = reads[rcv.read_idx];
            if (rd.status != SWEC_OK) continue;
            memcpy(rd.buf + rcv.buf_off, rcv.bufs[size_t(rcv.shard)].data(), rcv.len);
        }
    }
    return SWEC_OK;
}

}  // extern "C"

namespace {

// The needle parse of ScrubLocal (Needle.ReadBytes, needle_read.go:59-82), on the GPU.  The walk reads each record
// that is wholly local straight into a pinned slot of a staging ring, back to back at 8-byte alignment; a full slot
// goes H2D -> check kernels (needles.cu) -> results D2H on its own stream while the walk fills the next one.  A record
// larger than a slot gets a device buffer of its own.  Nothing touches the GPU until the first record arrives.
class NeedleScrub {
  public:
    NeedleScrub(int device, int version, uint32_t volume_id) : device_(device), version_(version), vid_(volume_id) {}
    ~NeedleScrub() { ring_.release(); }

    // room for the `bytes` of the next record: in the current slot (submitted first when it is full), or in a buffer
    // of its own when the record is larger than a slot
    int reserve(size_t bytes, uint8_t** out) {
        if (ring_.slots.empty()) {
            if (device_ < 0) return fail(SWEC_ERR_NO_DEVICE, "no CUDA device: the needle check runs on the GPU only");
            SWEC_CUDA(cudaSetDevice(device_));
            const int rc = ring_.allocate(device_, stage_slots(), kSlotData + kChecksBytes + needle_check_scratch_bytes(kSlotRecords));
            if (rc) return rc;
            pending_.resize(ring_.slots.size());
        }
        big_ = bytes > kSlotData;
        if (big_) {
            big_buf_.resize(bytes);
            *out = big_buf_.data();
            return SWEC_OK;
        }
        if (used_ + bytes > kSlotData || pending_[cur_].size() == kSlotRecords) {
            const int rc = submit();
            if (rc) return rc;
        }
        *out = ring_.slots[cur_].host + used_;
        return SWEC_OK;
    }

    // the record just read into the reserved room is whole: check it.  `finding` = its place among the findings.
    int commit(uint64_t id, int32_t size, size_t bytes, size_t finding) {
        swec_needle_check c{};
        c.needle_id = id;
        c.size = size;
        if (big_) return check_alone(c, bytes, finding);
        StagingSlot& s = ring_.slots[cur_];
        c.offset = int64_t(used_);
        checks(s.host)[pending_[cur_].size()] = c;
        pending_[cur_].push_back(finding);
        used_ += (bytes + 7) & ~size_t(7);
        return SWEC_OK;
    }

    int finish() {  // check what is still queued and collect every result
        int rc = submit();
        for (size_t i = 0; !rc && i < ring_.slots.size(); i++) rc = collect(i);
        return rc;
    }

    std::vector<std::pair<size_t, std::string>> failed;  // (finding, text) of every record that failed its check
    std::vector<swec_needle_check>* results = nullptr;   // when set: (*results)[finding] = every record's check

  private:
    static constexpr size_t kSlotData = size_t(16) << 20;  // record bytes per slot
    static constexpr int kSlotRecords = 16384;
    static constexpr size_t kChecksBytes = kSlotRecords * sizeof(swec_needle_check);
    static swec_needle_check* checks(uint8_t* slot_base) { return reinterpret_cast<swec_needle_check*>(slot_base + kSlotData); }

    int submit() {
        const size_t n = pending_.empty() ? 0 : pending_[cur_].size();
        if (n == 0) return SWEC_OK;
        StagingSlot& s = ring_.slots[cur_];
        const size_t cb = n * sizeof(swec_needle_check);
        SWEC_CUDA(cudaMemcpyAsync(s.dev, s.host, used_, cudaMemcpyHostToDevice, s.stream));
        SWEC_CUDA(cudaMemcpyAsync(checks(s.dev), checks(s.host), cb, cudaMemcpyHostToDevice, s.stream));
        SWEC_CUDA(launch_needle_check(s.dev, int64_t(used_), version_, checks(s.dev), int(n), s.dev + kSlotData + kChecksBytes, s.stream));
        SWEC_CUDA(cudaMemcpyAsync(checks(s.host), checks(s.dev), cb, cudaMemcpyDeviceToHost, s.stream));
        SWEC_CUDA(cudaEventRecord(s.done, s.stream));
        s.busy = true;
        used_ = 0;
        cur_ = (cur_ + 1) % ring_.slots.size();
        return collect(cur_);  // the next slot is reused: its results first
    }

    int collect(size_t i) {
        StagingSlot& s = ring_.slots[i];
        if (!s.busy) return SWEC_OK;
        SWEC_CUDA(cudaEventSynchronize(s.done));
        s.busy = false;
        const swec_needle_check* c = checks(s.host);
        for (size_t j = 0; j < pending_[i].size(); j++) note(c[j], pending_[i][j]);
        pending_[i].clear();
        return SWEC_OK;
    }

    int check_alone(swec_needle_check c, size_t bytes, size_t finding) {
        StagingSlot& s = ring_.slots[cur_];  // its stream; the slot's buffers stay with the walk
        const size_t at = (bytes + 7) & ~size_t(7);
        StreamScratch d(s.stream);
        SWEC_CUDA(d.alloc(at + sizeof c + needle_check_scratch_bytes(1)));
        auto* dc = reinterpret_cast<swec_needle_check*>(d.as<uint8_t>() + at);
        SWEC_CUDA(cudaMemcpyAsync(d.p, big_buf_.data(), bytes, cudaMemcpyHostToDevice, s.stream));
        SWEC_CUDA(cudaMemcpyAsync(dc, &c, sizeof c, cudaMemcpyHostToDevice, s.stream));
        SWEC_CUDA(launch_needle_check(d.p, int64_t(bytes), version_, dc, 1, dc + 1, s.stream));
        SWEC_CUDA(cudaMemcpyAsync(&c, dc, sizeof c, cudaMemcpyDeviceToHost, s.stream));
        SWEC_CUDA(cudaStreamSynchronize(s.stream));
        note(c, finding);
        return SWEC_OK;
    }

    void note(const swec_needle_check& c, size_t finding) {
        if (results) (*results)[finding] = c;
        std::string err;
        char buf[160];
        switch (c.status) {
            case SWEC_NEEDLE_OK: return;
            case SWEC_NEEDLE_SIZE_MISMATCH: err = "size mismatch"; break;  // ScrubLocal reads at offset 0: the short form
            case SWEC_NEEDLE_OUT_OF_RANGE:
                err = "index out of range " + std::to_string(c.range_index) + ": needle data corrupted";
                break;
            case SWEC_NEEDLE_BAD_CRC:  // %v of a NeedleId is hex (types/needle_id_type.go:34-36)
                snprintf(buf, sizeof buf, "invalid CRC for needle %" PRIx64 " (got %08x, want %08x), data on disk corrupted: needle data corrupted",
                         c.needle_id, c.crc_got, c.crc_want);
                err = buf;
                break;
            default: err = "record does not fit in its own bytes"; break;
        }
        failed.emplace_back(finding, "needle " + std::to_string(c.needle_id) + " on volume " + std::to_string(vid_) + ": " + err);
    }

    int device_, version_;
    uint32_t vid_;
    StagingRing ring_;
    std::vector<std::vector<size_t>> pending_;  // per slot: the finding index of each queued record
    size_t cur_ = 0, used_ = 0;
    bool big_ = false;
    std::vector<uint8_t> big_buf_;
};

// EcVolume.ScrubLocal (ec_volume_scrub.go:27-118): ScrubIndex, then every live entry of .ecx is located (GetActualSize
// ONCE here, unlike the read path) and each of its chunks read from the local shard that holds it.  A shard that is
// too short for a chunk, or cannot be read, is reported broken; chunks on shards that are not local are skipped like
// the reference skips remote ones.  With `needles`, every record whose chunks were all read is also checked like
// Needle.ReadBytes; its finding takes its place in walk order.
int scrub_walk(swec_ec_volume* v, NeedleScrub* needles, int64_t* entries, uint32_t* broken_shards, int* n_broken,
               char* errors, size_t errors_cap, int* n_errors) {
    if (!v || !entries || !n_broken || !n_errors || !broken_shards) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    std::lock_guard<std::mutex> lock(v->mu);
    std::vector<std::string> found;  // in walk order; "" = a record sent to the needle check
    int extra_lines = 0;
    {  // ScrubIndex = idx.CheckIndexFile on the sealed index
        int64_t n = 0;
        int k2 = 0;
        std::vector<char> buf(size_t(1) << 20);
        const int rc = swec_check_index_file((v->index_base + ".ecx").c_str(), v->version, &n, buf.data(), buf.size(), &k2);
        if (rc) return rc;
        if (k2) found.push_back(buf.data()), extra_lines = k2 - 1;
    }
    auto add = [&](const std::string& m) { found.push_back(m); };
    const int total = v->k + v->m;
    std::vector<int64_t> shard_size(size_t(total), -1);
    for (int i = 0; i < total; i++) {
        struct stat st;
        if (v->shard_fd[size_t(i)] >= 0 && fstat(v->shard_fd[size_t(i)], &st) == 0) shard_size[size_t(i)] = st.st_size;
    }
    std::vector<uint8_t> broken(size_t(total), 0), chunk;
    std::vector<Chunk> chunks;
    int64_t walked = 0;
    for (int64_t e = 0; e < v->entries(); e++) {
        walked++;
        const auto [id, offset, size] = v->entry(e);
        if (size == kTombstone) continue;  // Size.IsTombstone
        const int64_t want = needle_actual_size(size, v->version);
        if (const int rc = locate_chunks(v->shard_dat_size, v->k, offset, want, &chunks)) return rc;
        uint8_t* record = nullptr;  // where the record is gathered for the needle check, when all of it is local
        if (needles && size >= 0 &&
            std::all_of(chunks.begin(), chunks.end(), [&](const Chunk& c) { return v->shard_fd[size_t(c.shard)] >= 0; })) {
            const int rc = needles->reserve(size_t(want), &record);
            if (rc) return rc;
        }
        int64_t read = 0, pos = 0;
        for (size_t j = 0; j < chunks.size(); j++) {
            const auto [sid, soff, ssize] = chunks[j];
            const std::string where = std::to_string(j + 1) + "/" + std::to_string(chunks.size());
            uint8_t* dst = record ? record + pos : nullptr;
            pos += ssize;
            if (v->shard_fd[size_t(sid)] < 0) {  // not local: skipped, counted as read
                read += ssize;
                continue;
            }
            if (soff + ssize > shard_size[size_t(sid)]) {
                broken[size_t(sid)] = 1;
                add("local shard " + std::to_string(sid) + " for needle " + std::to_string(id) + " is too short (" +
                    std::to_string(shard_size[size_t(sid)]) + "), cannot read chunk " + where);
                continue;
            }
            if (!dst) {
                chunk.resize(size_t(ssize));
                dst = chunk.data();
            }
            const ssize_t got = pread(v->shard_fd[size_t(sid)], dst, size_t(ssize), off_t(soff));
            if (got < 0) {
                broken[size_t(sid)] = 1;
                add("failed to read chunk " + where + " for needle " + std::to_string(id) + " from local shard " + std::to_string(sid) +
                    " at offset " + std::to_string(soff) + ": " + strerror(errno));
                continue;
            }
            if (got != ssize) {
                broken[size_t(sid)] = 1;
                add("expected " + std::to_string(ssize) + " bytes for chunk " + where + " for needle " + std::to_string(id) +
                    " from local shard " + std::to_string(sid) + ", got " + std::to_string(got));
                continue;
            }
            read += got;
        }
        if (read != want) {  // the reference's walk stops here
            add("expected " + std::to_string(want) + " bytes for needle " + std::to_string(id) + ", got " + std::to_string(read));
            break;
        }
        if (record) {
            const int rc = needles->commit(id, size, size_t(want), found.size());
            if (rc) return rc;
            found.emplace_back();
        }
    }
    if (needles) {
        const int rc = needles->finish();
        if (rc) return rc;
        for (auto& [at, text] : needles->failed) found[at] = std::move(text);
    }
    std::string text;
    int count = extra_lines;
    for (const std::string& f : found) {
        if (f.empty()) continue;
        if (count++ > extra_lines) text += "\n";
        text += f;
    }
    *entries = walked;
    *n_broken = 0;
    for (int i = 0; i < total; i++)
        if (broken[size_t(i)]) broken_shards[(*n_broken)++] = uint32_t(i);
    *n_errors = count;
    copy_findings(text, errors, errors_cap);
    return SWEC_OK;
}

// The repair's re-check: every record of `named` (all its shards local) read from the shard files and checked the way
// scrub_needles checks a record.  (*out)[j] is the check of named[j], with its needle_id, offset and size; a record
// that runs past the end of its shard is SWEC_NEEDLE_OUTSIDE_IMAGE and is not checked.
int recheck_needles(swec_ec_volume* v, const std::vector<swec_needle_damage>& named, std::vector<swec_needle_check>* out) {
    out->assign(named.size(), swec_needle_check{});
    NeedleScrub scrub(v->device, v->version, 0);
    scrub.results = out;
    std::vector<Chunk> chunks;
    int rc;
    for (size_t j = 0; j < named.size(); j++) {
        const swec_needle_damage& r = named[j];
        const int64_t want = needle_actual_size(r.size, v->version);
        uint8_t* record = nullptr;
        if ((rc = locate_chunks(v->shard_dat_size, v->k, r.offset, want, &chunks)) || (rc = scrub.reserve(size_t(want), &record)))
            return rc;
        int64_t pos = 0;
        bool whole = true;
        for (const auto& [sid, soff, bytes] : chunks) {
            whole = whole && pread(v->shard_fd[size_t(sid)], record + pos, size_t(bytes), off_t(soff)) == ssize_t(bytes);
            pos += bytes;
        }
        if (!whole) (*out)[j].status = SWEC_NEEDLE_OUTSIDE_IMAGE;
        else if ((rc = scrub.commit(r.needle_id, r.size, size_t(want), j))) return rc;
    }
    if ((rc = scrub.finish())) return rc;
    for (size_t j = 0; j < named.size(); j++) {
        (*out)[j].needle_id = named[j].needle_id;
        (*out)[j].offset = named[j].offset;
        (*out)[j].size = named[j].size;
    }
    return SWEC_OK;
}

// The live records as the handle's reads see them: .ecx entries that are not deleted, minus the journalled ids
// (FindNeedleFromEcx, ec_volume.go:419-429), the journal re-read when it moved.  Under v->mu.
std::vector<swec_needle_damage> live_records(swec_ec_volume* v) {
    v->refresh_journal();
    std::vector<swec_needle_damage> recs;
    for (int64_t e = 0; e < v->entries(); e++) {
        const IndexEntry x = v->entry(e);
        if (size_deleted(x.size) || v->journalled(x.key)) continue;
        swec_needle_damage r{};
        r.needle_id = x.key;
        r.offset = x.offset;
        r.size = x.size;
        recs.push_back(r);
    }
    return recs;
}

// The named needles of the handle calls: the records with a non-zero count, in ascending needle id, left in *recs; the
// first needles_cap of them to needles[], how many there are to *n_needles.
void name_needles(std::vector<swec_needle_damage>* recs, swec_needle_damage* needles, int needles_cap, int* n_needles) {
    std::stable_sort(recs->begin(), recs->end(),
                     [](const swec_needle_damage& a, const swec_needle_damage& b) { return a.needle_id < b.needle_id; });
    recs->erase(std::remove_if(recs->begin(), recs->end(),
                               [](const swec_needle_damage& r) { return !r.damaged_bytes && !r.uncorrectable_bytes; }),
                recs->end());
    for (int j = 0; j < needles_cap && j < int(recs->size()); j++) needles[j] = (*recs)[size_t(j)];
    *n_needles = int(recs->size());
}

// Both needle damage calls on the handle (include/swec.h): every check before any device work, the live records as the
// reads see them, then pass 1 and, with damage, pass 2 (needle_damage_files).  With `checks` (the repair), pass 2 also
// writes the corrections, and every named needle is re-checked from the repaired files.
int handle_needle_damage(swec_ec_volume* v, int radius, const DamageOut& out, swec_needle_damage* needles, bool repair,
                         swec_needle_check* checks, int needles_cap, int* n_needles, uint64_t unowned[2], int* ok) {
    int rc = check_needle_damage_args(needles_cap, needles, unowned, 0, nullptr);
    if (rc) return rc;
    if (repair && needles_cap > 0 && !checks)
        return fail(SWEC_ERR_INVALID_ARG, "checks must be non-NULL when needles_cap is > 0");
    if (!v || !n_needles || !ok) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    std::lock_guard<std::mutex> lock(v->mu);
    if ((rc = out.check()) || (rc = check_radius(radius, 1, v->m))) return rc;
    *ok = 0;
    *n_needles = 0;
    unowned[0] = unowned[1] = 0;
    const int total = v->k + v->m;
    for (int i = 0; i < total; i++)
        if (v->shard_fd[size_t(i)] < 0)
            return fail(SWEC_ERR_TOO_FEW_SHARDS, std::string(repair ? "repairing" : "locating") +
                                                     " needle damage needs all shards; missing " + shard_ext(i));
    int64_t size = -1;
    for (int i = 0; i < total; i++)
        if ((rc = check_length(v->shard_fd[size_t(i)], &size))) return rc;
    if (v->device < 0) return fail(SWEC_ERR_NO_DEVICE, "no CUDA device: the volume was opened with device < 0");
    std::vector<swec_needle_damage> recs = live_records(v);
    if (!v->enc && (rc = swec_encoder_new(v->k, v->m, v->device, &v->enc))) return rc;
    const StripeMap map = StripeMap::locate(v->shard_dat_size, v->k, kLargeBlockSize, kSmallBlockSize);
    if ((rc = needle_damage_files(v->enc, v->shard_fd, size, radius, map, v->version, repair, &recs, out, unowned)))
        return rc;
    name_needles(&recs, needles, needles_cap, n_needles);
    if (!repair) {
        *ok = out.report->damaged_columns == 0 ? 1 : 0;
        return SWEC_OK;
    }
    std::vector<swec_needle_check> rechecked;
    if ((rc = recheck_needles(v, recs, &rechecked))) return rc;
    bool all_ok = out.report->uncorrectable_columns == 0;
    for (size_t j = 0; j < rechecked.size(); j++) {
        all_ok = all_ok && rechecked[j].status == SWEC_NEEDLE_OK;
        if (int(j) < needles_cap) checks[j] = rechecked[j];
    }
    *ok = all_ok ? 1 : 0;
    return SWEC_OK;
}

}  // namespace

extern "C" {

int swec_ec_volume_scrub_local(swec_ec_volume* v, int64_t* entries, uint32_t* broken_shards, int* n_broken, char* errors,
                               size_t errors_cap, int* n_errors) {
    return scrub_walk(v, nullptr, entries, broken_shards, n_broken, errors, errors_cap, n_errors);
}

int swec_ec_volume_scrub_needles(swec_ec_volume* v, uint32_t volume_id, int64_t* entries, uint32_t* broken_shards, int* n_broken,
                                 char* errors, size_t errors_cap, int* n_errors) {
    if (!v) return fail(SWEC_ERR_INVALID_ARG, "NULL volume");
    NeedleScrub needles(v->device, v->version, volume_id);
    return scrub_walk(v, &needles, entries, broken_shards, n_broken, errors, errors_cap, n_errors);
}

// what NewEcVolume derived from .vif and the shard files (ec_volume.go:114-154,399-417)
int swec_ec_volume_info(swec_ec_volume* v, int* data_shards, int* parity_shards, int* needle_version, int64_t* shard_dat_size,
                        uint32_t* local_shard_bits) {
    if (!v) return fail(SWEC_ERR_INVALID_ARG, "NULL volume");
    std::lock_guard<std::mutex> lock(v->mu);
    if (data_shards) *data_shards = v->k;
    if (parity_shards) *parity_shards = v->m;
    if (needle_version) *needle_version = v->version;
    if (shard_dat_size) *shard_dat_size = v->shard_dat_size;
    if (local_shard_bits) {
        uint32_t bits = 0;
        for (size_t i = 0; i < v->shard_fd.size(); i++)
            if (v->shard_fd[i] >= 0) bits |= 1u << i;
        *local_shard_bits = bits;
    }
    return SWEC_OK;
}

int swec_ec_volume_locate_needle_damage(swec_ec_volume* v, int radius, swec_damage_report* report, swec_damage_range* ranges,
                                        int ranges_cap, int* n_ranges, swec_needle_damage* needles, int needles_cap,
                                        int* n_needles, uint64_t unowned[2], int* ok) {
    return handle_needle_damage(v, radius, {report, ranges, ranges_cap, n_ranges}, needles, false, nullptr, needles_cap,
                                n_needles, unowned, ok);
}

int swec_ec_volume_repair_needle_damage(swec_ec_volume* v, int radius, swec_damage_report* report, swec_damage_range* ranges,
                                        int ranges_cap, int* n_ranges, swec_needle_damage* needles,
                                        swec_needle_check* checks, int needles_cap, int* n_needles, uint64_t unowned[2],
                                        int* ok) {
    return handle_needle_damage(v, radius, {report, ranges, ranges_cap, n_ranges}, needles, true, checks, needles_cap,
                                n_needles, unowned, ok);
}

int swec_ec_volume_sketch_needle_damage(swec_ec_volume* v, int64_t shard_len, const swec_sketch_page* pages,
                                        int64_t n_pages, swec_needle_damage* needles, int needles_cap, int* n_needles,
                                        uint64_t unowned[2]) {
    int rc = check_needle_damage_args(needles_cap, needles, unowned, 0, nullptr);
    if (rc) return rc;
    if (!v || !n_needles) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    if (shard_len < 0) return fail(SWEC_ERR_INVALID_ARG, "shard_len must be >= 0");
    if (n_pages < 0 || (n_pages > 0 && !pages))
        return fail(SWEC_ERR_INVALID_ARG, "n_pages must be >= 0, and pages non-NULL when it is > 0");
    std::lock_guard<std::mutex> lock(v->mu);
    if ((rc = check_sketch_pages(v->k, v->m, shard_len, pages, n_pages))) return rc;
    *n_needles = 0;
    unowned[0] = unowned[1] = 0;
    for (int fd : v->shard_fd) {  // a local shard of another length: the pages are not of this volume
        int64_t size = shard_len;
        if (fd >= 0 && (rc = check_length(fd, &size))) return rc;
    }
    if (n_pages == 0) return SWEC_OK;
    if (v->device < 0) return fail(SWEC_ERR_NO_DEVICE, "no CUDA device: the volume was opened with device < 0");
    std::vector<swec_needle_damage> recs = live_records(v);
    const StripeMap map = StripeMap::locate(v->shard_dat_size, v->k, kLargeBlockSize, kSmallBlockSize);
    if ((rc = sketch_needle_damage(v->device, map, shard_len, pages, n_pages, recs.data(), int(recs.size()), v->version,
                                   unowned)))
        return rc;
    name_needles(&recs, needles, needles_cap, n_needles);
    return SWEC_OK;
}

int swec_ec_volume_page_sketch(swec_ec_volume* v, uint64_t seed, uint64_t* const* sketches, int64_t sketches_cap,
                               int64_t* shard_len, int64_t* n_pages) {
    if (!v || !sketches || !shard_len || !n_pages) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    if (sketches_cap < 0) return fail(SWEC_ERR_INVALID_ARG, "sketches_cap must be >= 0");
    std::lock_guard<std::mutex> lock(v->mu);
    std::vector<int> fds;
    std::vector<uint64_t*> out;
    for (int i = 0; i < v->k + v->m; i++) {
        if (!sketches[i]) continue;
        if (v->shard_fd[size_t(i)] < 0) return fail(SWEC_ERR_TOO_FEW_SHARDS, "shard " + shard_ext(i) + " is not local");
        fds.push_back(v->shard_fd[size_t(i)]);
        out.push_back(sketches[i]);
    }
    if (fds.empty()) return fail(SWEC_ERR_INVALID_ARG, "no shard requested: every sketches entry is NULL");
    int64_t size = -1;
    int rc;
    for (int fd : fds)
        if ((rc = check_length(fd, &size))) return rc;
    if (size > 0) {
        if (v->device < 0) return fail(SWEC_ERR_NO_DEVICE, "no CUDA device: the volume was opened with device < 0");
        if (!v->enc && (rc = swec_encoder_new(v->k, v->m, v->device, &v->enc))) return rc;
        if ((rc = page_sketch_files(v->enc, fds, size, seed, out.data(), sketches_cap))) return rc;
    }
    *shard_len = size;
    *n_pages = (size + 4095) / 4096;
    return SWEC_OK;
}

// FileAndDeleteCount (ec_volume.go:330-349): entries of the sealed .ecx, and distinct journalled ids.
int swec_ec_volume_counts(swec_ec_volume* v, uint64_t* file_count, uint64_t* delete_count) {
    if (!v) return fail(SWEC_ERR_INVALID_ARG, "NULL volume");
    std::lock_guard<std::mutex> lock(v->mu);
    v->refresh_journal();
    if (file_count) *file_count = uint64_t(v->entries());
    if (delete_count) *delete_count = uint64_t(v->deleted.size());
    return SWEC_OK;
}

// DeleteNeedleFromEcx (ec_volume_delete.go:28-93): .ecx stays sealed; a runtime delete appends the id to the
// .ecj journal (the durable commit point: written, fsync'ed, truncated back on failure) and only then becomes
// visible to reads.  Unknown ids and ids that are already tombstoned / journalled are not errors.
int swec_ec_volume_delete_needle(swec_ec_volume* v, uint64_t needle_id) {
    if (!v) return fail(SWEC_ERR_INVALID_ARG, "NULL volume");
    std::lock_guard<std::mutex> lock(v->mu);
    const int64_t found = v->find(needle_id);
    if (found < 0) return SWEC_OK;                          // already gone
    if (size_deleted(v->entry(found).size)) return SWEC_OK;  // folded into .ecx by an earlier rebuild
    // the in-memory set is authoritative between external changes of the file (refresh_journal notices those by
    // size / mtime / inode): an O(log n) membership test and an 8-byte append per delete, like the reference's map
    // check + append — not a re-read of the whole journal
    v->refresh_journal();
    if (v->journalled(needle_id)) return SWEC_OK;  // idempotent
    const std::string path = v->index_base + ".ecj";
    const int fd = open(path.c_str(), O_WRONLY | O_CREAT, 0644);
    if (fd < 0) return fail(SWEC_ERR_IO, "cannot open ec volume journal " + path + ": " + strerror(errno));
    struct stat st;
    if (fstat(fd, &st) != 0) {
        const int e = errno;
        close(fd);
        return fail(SWEC_ERR_IO, "stat ecj: " + std::string(strerror(e)));
    }
    uint8_t b[8];
    put_be64(b, needle_id);
    const bool ok = pwrite(fd, b, 8, st.st_size) == 8 && fsync(fd) == 0;
    const int e = errno;
    if (!ok) {
        if (ftruncate(fd, st.st_size) != 0) {}  // keep journal and in-memory state from drifting
        close(fd);
        return fail(SWEC_ERR_IO, "write ecj: " + std::string(strerror(e)));
    }
    struct stat after;
    const bool stat_ok = fstat(fd, &after) == 0;
    close(fd);
    v->deleted.insert(std::upper_bound(v->deleted.begin(), v->deleted.end(), needle_id), needle_id);
    v->ecj_seen = stat_ok ? swec_ec_volume::stamp(&after) : swec_ec_volume::JournalStamp{};  // else re-read on the next use
    return SWEC_OK;
}

int swec_read_ec_needles(const char* data_base, const char* index_base, const char* const* additional_dirs,
                         int n_additional_dirs, swec_needle_read* reads, int n_reads, int device) {
    if (n_reads > 0 && !reads) return fail(SWEC_ERR_INVALID_ARG, "NULL argument");
    swec_ec_volume* v = nullptr;
    int rc = swec_ec_volume_open(data_base, index_base, additional_dirs, n_additional_dirs, device, &v);
    if (rc) return rc;
    rc = swec_ec_volume_read_needles(v, reads, n_reads);
    swec_ec_volume_close(v);
    return rc;
}

}  // extern "C"
