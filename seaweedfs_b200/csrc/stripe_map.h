// seaweedfs_b200/csrc/stripe_map.h — the inverse of the two-tier striping, stated once for host and device code:
// byte x of data shard i -> its offset in the .dat.  Two geometries share the formula and differ only in how many rows
// of large blocks there are:
//   encode   the striping encodeDatFile writes (ec_encoder.go:280-321, StripeGeometry in volume_format.h): large rows
//            while a whole large row of the .dat remains, then small rows; the zero padding of the last row, and
//            anything past it, is no .dat byte at all
//   locate   the striping LocateData reads (ec_locate.go:16-98, swec_locate_data): shard_dat_size / large rows of
//            large blocks, then small rows without end
// needle_damage.cu maps located bytes to needles with it, sketch.cu the runs of flagged pages; the host only builds
// the map.
#pragma once
#include <cstdint>

#include "needle_format.h"  // SWEC_HD

namespace swec {

struct StripeMap {
    int64_t large, small;
    int64_t large_rows;  // rows of k large blocks
    int64_t dat_end;     // .dat offsets at or past it are padding (INT64_MAX: no bound)
    int k;

    static StripeMap encode(int64_t dat_size, int k, int64_t large, int64_t small) {
        return {large, small, dat_size / (large * k), dat_size, k};
    }
    static StripeMap locate(int64_t shard_dat_size, int k, int64_t large, int64_t small) {
        return {large, small, shard_dat_size / large, INT64_MAX, k};
    }

    // the .dat offset of byte x of data shard i, or -1 when that byte is padding
    SWEC_HD int64_t dat_offset(int i, int64_t x) const {
        const int64_t large_bytes = large_rows * large;  // of every shard
        int64_t d;
        if (x < large_bytes) {
            d = (x / large) * large * k + int64_t(i) * large + x % large;
        } else {
            const int64_t y = x - large_bytes;
            d = large_bytes * k + (y / small) * small * k + int64_t(i) * small + y % small;
        }
        return d < dat_end ? d : -1;
    }

    // the shard offset where the block holding shard offset x ends: in every data shard, the bytes [x, block_end(x))
    // have consecutive .dat offsets (until those reach dat_end)
    SWEC_HD int64_t block_end(int64_t x) const {
        const int64_t large_bytes = large_rows * large;
        if (x < large_bytes) return (x / large + 1) * large;
        return large_bytes + ((x - large_bytes) / small + 1) * small;
    }
};

}  // namespace swec
