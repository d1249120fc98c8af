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
