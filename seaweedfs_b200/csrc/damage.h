// seaweedfs_b200/csrc/damage.h — which shard is wrong, from the parity syndrome of every byte column (damage.cu), for
// the file pipeline (ec_files.cc) and the device-level calls (engine.cc); optionally corrected in place.
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
    bool correcting() const { return correct_; }
    // Columns [base, base + n) of the set: computed[p] is the parity re-encoded from the data shards, shards[0..k+m) the
    // shards as found (stored parity at shards[k+p]).  The shards are only read unless correcting; a correcting launch
    // must come after the encode that read the data shards, in stream order.  Asynchronous on `s`.
    int launch(const uint8_t* const* computed, uint8_t* const* shards, size_t n, int64_t base, cudaStream_t s);
    // After every launch has completed: the report, the page ranges (first ranges_cap of them) and their total; `all`
    // (may be NULL) receives every range.
    int collect(swec_damage_report* report, swec_damage_range* ranges, int ranges_cap, int* n_ranges,
                std::vector<swec_damage_range>* all = nullptr);

  private:
    int k_ = 0, m_ = 0, radius_ = 1;
    bool correct_ = false;
    int64_t shard_len_ = 0;
    size_t page_words_ = 0;  // 32-bit words of one page bitmap
    uint32_t* tables_ = nullptr;
    unsigned long long* counters_ = nullptr;
    uint32_t* pages_ = nullptr;
};

}  // namespace swec
