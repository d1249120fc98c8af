// seaweedfs_b200/csrc/damage.h — which shard is wrong, from the parity syndrome of every byte column (damage.cu), for
// the file pipeline (ec_files.cc) and the device-level calls (engine.cc); optionally corrected in place, or carried into
// the shards a rebuild computes.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/swec.h"
#include "gf256.h"

namespace swec {

// The argument rules every entry point shares: radius 1 needs m >= 2 and radius 2 needs m >= 4, a report is required,
// ranges_cap must not be negative and ranges may only be NULL when ranges_cap is 0.
int check_locate_args(int m, int radius, const swec_damage_report* report, const swec_damage_range* ranges,
                      int ranges_cap);
// The checked rebuild's rules: those of check_locate_args without the parity count, and radius 0, 1 or 2 (clamped to
// what the present shards allow by DamageLocator::init_rebuild).
int check_rebuild_args(int radius, const swec_damage_report* report, const swec_damage_range* ranges, int ranges_cap);
// The report of a set where nothing could be checked: no columns, no shards, no ranges (n_ranges may be NULL).
void unchecked_report(swec_damage_report* report, int* n_ranges);
// ec.decode's plan from rs_reconstruct_plan's: the entries of `outs` that are missing parity shards, and their rows of
// `fused`, removed, so that one apply rebuilds only the missing data shards and re-encodes the present check shards.
void drop_missing_parity(const uint8_t* present, int k, std::vector<int>* outs, Matrix* fused);

// Accumulates, over any number of launches, the shards blamed for every byte column of a shard set whose syndrome
// (computed parity XOR stored parity) is not zero.  Device memory lives on the device current at init().
class DamageLocator {
  public:
    DamageLocator() = default;
    DamageLocator(const DamageLocator&) = delete;
    DamageLocator& operator=(const DamageLocator&) = delete;
    ~DamageLocator();

    // parity: the m x k parity rows of the code.  correct: every launch also replaces the blamed bytes of the columns it
    // decodes within the radius by their decoded values.  Clears the counters on `s` and synchronises it.
    int init(const Matrix& parity, int64_t shard_len, int radius, cudaStream_t s, bool correct = false);
    // Errors and erasures: a set whose shards `outs` are rebuilt or re-encoded from the information set `info` (the
    // first k present shards, ascending) by the rows of `fused` (one per entry of `outs`, ascending ids, as
    // rs_reconstruct_plan gives them for a mask of `info` alone).  The present ones among `outs` (c >= 1 of them) are the
    // check shards; the code punctured to info + check has distance c+1, so the radius is clamped to c/2, and 0
    // decodes nothing.  Launches also take the errors of the information shards they locate out of the missing shards'
    // rows.  The report and ranges name shard ids; check ids exceed information ids, so ranges stay in ascending id.
    // decode: `outs` holds only missing data shards and check shards (every check shard is then a parity shard), and
    // launches also correct the errors they locate in information shards that are data shards, in place.
    int init_rebuild(const Matrix& fused, const std::vector<int>& info, const std::vector<int>& outs,
                     const uint8_t* present, int64_t shard_len, int radius, cudaStream_t s, bool decode = false);
    bool correcting() const { return correct_; }
    // Columns [base, base + n) of the set: computed[p] is the parity re-encoded from the data shards, shards[0..k+m) the
    // shards as found (stored parity at shards[k+p]).  The shards are only read unless correcting; a correcting launch
    // must come after the encode that read the data shards, in stream order.  Asynchronous on `s`.
    // Rebuild mode: computed[o] is row o of `fused`, shards[0..k) the information shards and shards[k..k+c) the check
    // shards in ascending id; only the rows of missing shards in `computed` are written, after the apply that made them.
    // Decode mode also writes shards[j] of the information shards that are data shards.
    int launch(uint8_t* const* computed, uint8_t* const* shards, size_t n, int64_t base, cudaStream_t s);
    // After every launch has completed: the report, the page ranges (first ranges_cap of them) and their total; `all`
    // (may be NULL) receives every range.
    int collect(swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges,
                std::vector<swec_damage_range>* all = nullptr);

  private:
    int k_ = 0, m_ = 0, radius_ = 1;  // m_: check positions (c in rebuild mode)
    bool correct_ = false, rebuild_ = false, decode_ = false;
    std::vector<int> ids_;                   // shard id of every kernel position, ascending
    std::vector<int> check_rows_, out_rows_;  // rebuild mode: rows of `computed` that are check shards / rebuilt shards
    int64_t shard_len_ = 0;
    size_t page_words_ = 0;  // 32-bit words of one page bitmap
    uint32_t* tables_ = nullptr;
    unsigned long long* counters_ = nullptr;
    uint32_t* pages_ = nullptr;
    uint32_t* rtables_ = nullptr;  // rebuild mode: log R
};

}  // namespace swec
