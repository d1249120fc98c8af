// seaweedfs_b200/csrc/damage.h — which shard is wrong, from the parity syndrome of every byte column (damage.cu), for
// the file pipeline (ec_files.cc) and the device-level calls (engine.cc); optionally corrected in place, or carried into
// the shards a rebuild computes.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/swec.h"
#include "engine.h"
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

// Errors and erasures over a presence mask: the first k present shards are the information set, and one apply of
// `fused` computes every other shard in `outs` from it; the present ones are the check shards, the missing ones are
// rebuilt.  With every shard present, the information set is the data shards and the checks are the parity shards.
struct CheckedPlan {
    std::vector<int> info;          // the first k present shards, ascending
    std::vector<int> outs;          // every other shard the apply computes, ascending; decode: no missing parity shard
    Matrix fused;                   // row o computes outs[o] from the information shards
    std::vector<int> check_rows;    // the entries of `outs` that are present, ascending
    std::vector<int> rebuilt_rows;  // the entries of `outs` that are missing, ascending
    bool decode = false;            // ec.decode: only the missing data shards are rebuilt

    bool build(const Matrix& gen, int k, const uint8_t* present, bool decode);  // false: fewer than k present
    int c() const { return int(check_rows.size()); }
    int check(int i) const { return outs[size_t(check_rows[size_t(i)])]; }      // shard id of check shard i
    int rebuilt(int r) const { return outs[size_t(rebuilt_rows[size_t(r)])]; }  // shard id of rebuilt shard r
    // The locator's position of shard `id`, which the file pipeline's slot streams and the device loop's shard arrays
    // share: information shard j at j, check shard i at k+i, computed row o at k+c+o; -1 for any other shard.
    int position(int id) const;
};

// Accumulates, over any number of launches, the shards blamed for every byte column of a shard set whose syndrome
// (computed parity XOR stored parity) is not zero.  Device memory lives on the device current at init().
class DamageLocator {
  public:
    DamageLocator() = default;
    DamageLocator(const DamageLocator&) = delete;
    DamageLocator& operator=(const DamageLocator&) = delete;

    // parity: the m x k parity rows of the code.  correct: every launch also replaces the blamed bytes of the columns it
    // decodes within the radius by their decoded values.  Clears the counters on `s` and synchronises it.
    int init(const Matrix& parity, int64_t shard_len, int radius, cudaStream_t s, bool correct = false);
    // Errors and erasures over `plan`, which has c >= 1 check shards: the code punctured to information + check shards
    // has distance c+1, so the radius is clamped to c/2, and 0 decodes nothing.  Launches also take the errors of the
    // information shards they locate out of the rebuilt rows.  The report and ranges name shard ids; check ids exceed
    // information ids, so ranges stay in ascending id.  plan.decode (every check shard is then a parity shard):
    // launches also correct the errors they locate in information shards that are data shards, in place.
    int init_rebuild(const CheckedPlan& plan, int64_t shard_len, int radius, cudaStream_t s);
    bool correcting() const { return correct_; }
    // Columns [base, base + n) of the set: computed[p] is the parity re-encoded from the data shards, shards[0..k+m) the
    // shards as found (stored parity at shards[k+p]).  The shards are only read unless correcting; a correcting launch
    // must come after the encode that read the data shards, in stream order.  Asynchronous on `s`.
    // Rebuild mode: computed[o] is row o of the plan's `fused`, shards[0..k+c) the information and check shards at
    // their positions; only the rebuilt rows in `computed` are written, after the apply that made them.
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
    DeviceBuffer tables_;    // LocateTables
    DeviceBuffer counters_;  // unsigned long long: bytes, first and last of every set, damaged columns
    DeviceBuffer pages_;     // uint32_t: one page bitmap per set
    DeviceBuffer rtables_;   // rebuild mode: RebuildTables (log R)
};

}  // namespace swec
