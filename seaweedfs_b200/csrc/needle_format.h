// seaweedfs_b200/csrc/needle_format.h — the needle record of a SeaweedFS volume, stated once for host and device code:
//   header: cookie 4, id 8, Size 4, big-endian              weed/storage/needle/needle.go, needle_read.go:102-106
//   body (v2/v3): DataSize 4, Data, Flags 1, name / mime / last-modified / TTL / pairs by flag
//                                                          needle_read.go:108-181
//   tail: checksum 4 (+ append timestamp 8 in v3), padding to 8   needle_read_tail.go:11-50
// The host only hands (offset, Size) entries to the GPU and computes record extents with needle_actual_size; the walk
// through the body (record_layout) runs in the check kernel (needles.cu).  No CRC here.
#pragma once
#include <cstdint>

#include "../../include/swec.h"

#if defined(__CUDACC__)
#define SWEC_HD __host__ __device__ __forceinline__
#else
#define SWEC_HD inline
#endif

namespace swec {

constexpr int kNeedleHeaderSize = 16;  // NeedleHeaderSize: cookie + id + Size
constexpr int kNeedleIdOffset = 4, kNeedleSizeOffset = 12;
constexpr int kNeedleChecksumSize = 4, kTimestampSize = 8, kNeedlePaddingSize = 8;
constexpr int kDataSizeSize = 4, kLastModifiedSize = 5, kTtlSize = 2, kPairsSizeSize = 2;
// Flags (needle_read.go:16-22)
constexpr uint8_t kFlagHasName = 0x02, kFlagHasMime = 0x04, kFlagHasLastModified = 0x08, kFlagHasTtl = 0x10,
                  kFlagHasPairs = 0x20;

// GetActualSize (needle/needle_read.go:292-294, needle_read_tail.go:36-50): header 16 + body + checksum 4
// (+ 8-byte timestamp in version 3) + padding to 8, where the padding is 1..8 bytes, never 0.
SWEC_HD int64_t needle_actual_size(int64_t size, int version) {
    const int64_t fixed = kNeedleHeaderSize + size + kNeedleChecksumSize + (version == 3 ? kTimestampSize : 0);
    return fixed + (kNeedlePaddingSize - fixed % kNeedlePaddingSize);
}

SWEC_HD uint32_t needle_be32(const uint8_t* p) {
    return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3];
}

struct RecordLayout {
    int32_t status;       // SWEC_NEEDLE_OK (go on to the CRC), SWEC_NEEDLE_SIZE_MISMATCH or SWEC_NEEDLE_OUT_OF_RANGE
    int32_t range_index;  // 1..7 with SWEC_NEEDLE_OUT_OF_RANGE: which bound of readNeedleDataVersion2 failed
    uint32_t data_size;   // bytes of Data
    int32_t data_offset;  // where Data starts, from the record's first byte
    uint32_t crc_want;    // the checksum stored after the body
};

// Needle.ReadBytes(rec, 0, size, version) up to the CRC (needle_read.go:59-82,108-181): the header Size must equal the
// index Size, then (v2/v3) DataSize and every optional field must stay inside the body.  `rec` holds at least
// needle_actual_size(size, version) bytes.
SWEC_HD RecordLayout record_layout(const uint8_t* rec, int32_t size, int version) {
    RecordLayout r{SWEC_NEEDLE_OK, 0, 0, kNeedleHeaderSize, 0};
    if (int32_t(needle_be32(rec + kNeedleSizeOffset)) != size || size < 0) {
        r.status = SWEC_NEEDLE_SIZE_MISMATCH;
        return r;
    }
    r.crc_want = needle_be32(rec + kNeedleHeaderSize + size);
    if (version == 1) {  // Data is the whole body
        r.data_size = uint32_t(size);
        return r;
    }
    const uint8_t* b = rec + kNeedleHeaderSize;
    const int64_t len = size;
    int64_t i = 0;
    auto out_of_range = [&](int which) {
        r.status = SWEC_NEEDLE_OUT_OF_RANGE;
        r.range_index = which;
        r.data_size = 0;
        return r;
    };
    if (i < len) {  // a body of 1..3 bytes cannot hold DataSize: the bound below fails, as in the reference
        const uint32_t ds = needle_be32(b);
        i += kDataSizeSize;
        if (int64_t(ds) + i > len) return out_of_range(1);
        r.data_size = ds;
        r.data_offset = kNeedleHeaderSize + kDataSizeSize;
        i += ds;
    }
    uint8_t flags = 0;
    if (i < len) flags = b[i++];
    if (i < len && (flags & kFlagHasName)) {
        const int64_t n = b[i++];
        if (n + i > len) return out_of_range(2);
        i += n;
    }
    if (i < len && (flags & kFlagHasMime)) {
        const int64_t n = b[i++];
        if (n + i > len) return out_of_range(3);
        i += n;
    }
    if (i < len && (flags & kFlagHasLastModified)) {
        if (kLastModifiedSize + i > len) return out_of_range(4);
        i += kLastModifiedSize;
    }
    if (i < len && (flags & kFlagHasTtl)) {
        if (kTtlSize + i > len) return out_of_range(5);
        i += kTtlSize;
    }
    if (i < len && (flags & kFlagHasPairs)) {
        if (kPairsSizeSize + i > len) return out_of_range(6);
        const int64_t n = (int64_t(b[i]) << 8) | b[i + 1];
        i += kPairsSizeSize;
        if (n + i > len) return out_of_range(7);
    }
    return r;
}

}  // namespace swec
