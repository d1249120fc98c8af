// seaweedfs_b200/csrc/needle_damage.h — which needles the located damage hits (needle_damage.cu), for the device call
// and the mounted volume's file-level call (ec_files.cc, ec_volume.cc).
//
// Per piece of columns: a copy of the data shards as found, the correcting locate on the piece, the corrected data
// re-encoded; then one kernel classifies every column of every data shard (damaged: the corrected byte differs from the
// one found; uncorrectable: the column's residual syndrome, re-encoded parity XOR corrected parity, is not zero) and adds
// each such byte to the live record that owns its .dat offset, or to the unowned counters.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/swec.h"
#include "damage.h"
#include "engine.h"
#include "stripe_map.h"

namespace swec {

// The new argument rules of both needle damage calls, checked before any other.
int check_needle_damage_args(int needles_cap, const swec_needle_damage* needles, const uint64_t* unowned,
                             int n_records, const swec_needle_damage* records);

// The live records in device memory, sorted by offset, and their counters: what the attribution kernels add to
// (needle_damage.cu per byte, sketch.cu per run of a flagged page).  The ownership rule lives here alone: a .dat byte
// belongs to the record with the greatest offset not above it (the later entry on a tie) when it lies inside it.
struct RecordTally {
    const int64_t* off;  // [n], ascending
    const int64_t* end;  // [n]
    int n;
    unsigned long long* damaged;        // [n]
    unsigned long long* uncorrectable;  // [n]
    unsigned long long* unowned;        // [2]
    unsigned* mask;                     // [n]

    // the last record whose offset is not above d, or -1: the only one that can own d
    SWEC_HD int candidate(int64_t d) const {
        int lo = 0, hi = n;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (off[mid] <= d) lo = mid + 1;
            else hi = mid;
        }
        return lo - 1;
    }
    // the record that owns .dat offset d (-1 for none, and for padding, d < 0)
    SWEC_HD int owner(int64_t d) const {
        if (d < 0) return -1;
        const int p = candidate(d);
        return p >= 0 && d < end[p] ? p : -1;
    }
    // how many bytes of [lo, hi) record p owns, p = candidate(x) for some x in [lo, hi): the candidate of a byte
    // stays p up to the next record's offset
    SWEC_HD int64_t owned(int p, int64_t lo, int64_t hi) const {
        int64_t stop = end[p] < hi ? end[p] : hi;
        if (p + 1 < n && off[p + 1] < stop) stop = off[p + 1];
        const int64_t start = off[p] > lo ? off[p] : lo;
        return stop > start ? stop - start : 0;
    }
};

class NeedleDamage {
  public:
    NeedleDamage() = default;
    NeedleDamage(const NeedleDamage&) = delete;
    NeedleDamage& operator=(const NeedleDamage&) = delete;

    // recs[n]: every live record (offset and size read; any order).  A record owns [offset, offset +
    // needle_actual_size(size, version)); of overlapping records, a byte belongs to the one with the greatest offset not
    // above it (the later entry on a tie) when it lies inside that record.  `slots` pieces of up to `piece` columns get
    // scratch for a copy of their data shards.  Device memory lives on the current device; synchronises `s`.
    int init(int k, int m, const StripeMap& map, const swec_needle_damage* recs, int n, int version, int slots,
             size_t piece, cudaStream_t s);
    // the slot's copy of the piece's data shards, taken before the correcting locate writes them
    int save(uint8_t* const* shards, size_t len, int slot, cudaStream_t s);
    // Columns [base, base + len): orig[k] the data shards as found (NULL: the slot's saved copy), fixed[k+m] the shards
    // after the correcting locate, comp[m] the parity re-encoded from fixed[0..k).  Asynchronous on `s`.
    int launch(const uint8_t* const* orig, uint8_t* const* fixed, uint8_t* const* comp, size_t len, int64_t base,
               int slot, cudaStream_t s);
    // after every launch has completed: shard_mask, damaged_bytes and uncorrectable_bytes of recs[n] (init's order)
    int collect(swec_needle_damage* recs, uint64_t unowned[2]);
    // the sorted records and counters, for a kernel of another translation unit (sketch.cu); after init
    RecordTally tally() const;

  private:
    int k_ = 0, m_ = 0, n_ = 0;
    StripeMap map_{};
    size_t piece_ = 0;
    std::vector<int> order_;                 // sorted position -> index in recs
    DeviceBuffer spans_;     // int64_t offset[n], end[n], sorted by offset
    DeviceBuffer counters_;  // unsigned long long damaged[n], uncorrectable[n], unowned[2]
    DeviceBuffer masks_;     // unsigned [n]
    DeviceBuffer saved_;     // slots x k x piece bytes
};

// The file work of the handle's needle damage calls (ec_files.cc) on the k+m local shard files `in`, all `size` bytes:
// pass 1 is the locate pass of swec_locate_ec_damage; when it finds damage, pass 2 reads the flagged pages again, as
// the repair does, through a NeedleDamage over `recs` mapped by `map`.  recs' counts and unowned are left zero on a
// clean set.  `repair`: pass 2 also writes what swec_repair_ec_damage's pass 2 writes, to the files behind `in`.
int needle_damage_files(swec_encoder* enc, const std::vector<int>& in, int64_t size, int radius, const StripeMap& map,
                        int version, bool repair, std::vector<swec_needle_damage>* recs, const DamageOut& out,
                        uint64_t unowned[2]);

}  // namespace swec
