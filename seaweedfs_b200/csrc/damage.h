// seaweedfs_b200/csrc/damage.h — which shard is wrong, from the parity syndrome of every byte column (damage.cu), for
// the file pipeline (ec_files.cc) and the device-level calls (engine.cc); optionally corrected in place, or carried into
// the shards a rebuild computes.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/swec.h"
#include "engine.h"
#include "gf256.h"

namespace swec {

// The report out-parameters of every damage call: the report, the first `cap` page ranges and their total.
struct DamageOut {
    swec_damage_report* report;
    swec_damage_range* ranges;
    int cap;
    int* n_ranges;         // may be NULL
    bool checked = false;  // the checked file calls: set once the report comes from a locator (c >= 1)

    // a report is required, cap must not be negative and ranges may only be NULL when cap is 0
    int check() const;
    // the report of a set where nothing could be checked: no columns, no shards, no ranges
    void unchecked() const;
};

// The radius rule: `lowest` (0 or 1) up to 2, and radius t needs 2t <= m parity shards (the default m sets no bound:
// the checked calls clamp the radius to what their present shards allow, CheckedPlan::radius).
int check_radius(int radius, int lowest, int m = INT_MAX);

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
    // every shard present: the data shards are the information set, fused is the parity rows, the checks are parity
    static CheckedPlan all_present(const Matrix& gen, int k);
    int c() const { return int(check_rows.size()); }
    int check(int i) const { return outs[size_t(check_rows[size_t(i)])]; }      // shard id of check shard i
    int rebuilt(int r) const { return outs[size_t(rebuilt_rows[size_t(r)])]; }  // shard id of rebuilt shard r
    // The locator's position of shard `id`, which the file pipeline's slot streams and the device loop's shard arrays
    // share: information shard j at j, check shard i at k+i, computed row o at k+c+o; -1 for any other shard.
    int position(int id) const;

    // What the locate kernel and the sketch page decode both read of the code punctured to the information and check
    // shards, which has distance c+1:
    Matrix checks() const;  // P', the c x k rows of `fused` that compute the check shards
    // log R[r][j] of rebuilt row r at byte r*32 + j of kLogRBytes, kLogZero for a zero entry (locate_decode.cuh)
    void rebuilt_logs(uint8_t* logr) const;
    int radius(int t) const { return std::min(t, c() / 2); }  // radius t needs 2t <= c
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
    // After every launch has completed: the report, the page ranges (the first out.cap of them) and their total; `all`
    // (may be NULL) receives every range.
    int collect(const DamageOut& out, std::vector<swec_damage_range>* all = nullptr);

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
