// seaweedfs_b200/csrc/locate_decode.cuh — the column decoder of the locate kernels (damage.cu), shared with the page
// decode of the sketch calls (sketch.cu): which <= radius shards explain a non-zero parity syndrome, against log/exp
// tables and the logs of P in shared memory.  damage.cu states the cases it decodes.
#pragma once
#include <cuda_runtime.h>

#include <cstring>

#include "apply_params.h"
#include "gf256.h"

namespace swec {

namespace {

struct LocateTables {
    u8 log[256];
    u8 exp[512];         // two periods of 2^i: a sum of two logs needs no reduction
    u8 logp[32 * 32];    // log P[i][j] at i*32 + j
    u8 logdet[32 * 32];  // log det [P0a P0b; P1a P1b] at a*32 + b (a != b data shards)
};
constexpr int kTableWords = int(sizeof(LocateTables) / 4);
static_assert(sizeof(LocateTables) % 16 == 0, "tables are copied in words");

// The log R table of the rebuilding decodes (CheckedPlan::rebuilt_logs): log R[r][j] of rebuilt row r and information
// position j at byte r*32 + j, kLogZero for a zero entry (logs of non-zero bytes are < 255).
constexpr u8 kLogZero = 0xff;
constexpr int kLogRBytes = 32 * 32;
constexpr int kLogRWords = kLogRBytes / 4;

// logs of the field's non-zero bytes (to base 2), and two periods of powers of 2
void log_exp_tables(u8* log, u8* exp) {
    unsigned x = 1;
    for (int i = 0; i < 255; i++) {
        exp[i] = u8(x);
        log[x] = u8(i);
        x <<= 1;
        if (x & 0x100) x ^= kFieldPoly;
    }
    for (int i = 255; i < 512; i++) exp[i] = exp[i - 255];
}

// the tables decode_column reads, for the code with these m x k parity rows
void locate_tables(const Matrix& parity, LocateTables* t) {
    const int k = parity.cols, m = parity.rows;
    memset(t, 0, sizeof *t);
    log_exp_tables(t->log, t->exp);
    const GF& gf = GF::get();
    for (int i = 0; i < m; i++)
        for (int j = 0; j < k; j++) t->logp[i * 32 + j] = t->log[parity.at(i, j)];
    for (int a = 0; a < k && m >= 2; a++)
        for (int b = 0; b < k; b++)
            if (a != b)
                t->logdet[a * 32 + b] = t->log[gf.mul[parity.at(0, a)][parity.at(1, b)] ^ gf.mul[parity.at(0, b)][parity.at(1, a)]];
}

__device__ __forceinline__ u8 gmul(const LocateTables& t, int log_c, u8 v) { return v ? t.exp[log_c + t.log[v]] : 0; }

// rows other than `skip` of s (logs in L, all non-zero) are one multiple of column j of P; r is the log of that
// multiple, the error value of data shard j
__device__ __forceinline__ bool multiple_of_column(const LocateTables& t, const u8* L, int m, int j, int skip, int& r) {
    r = -1;
    for (int i = 0; i < m; i++) {
        if (i == skip) continue;
        int d = int(L[i]) - int(t.logp[i * 32 + j]);
        if (d < 0) d += 255;
        if (r < 0) r = d;
        else if (d != r) return false;
    }
    return true;
}

// Shards that explain the non-zero syndrome s within the radius, ascending in *a, *b; returns how many (0: none does).
// VALUES: also their error values in *ea, *eb, the bytes that XORed into the shards turn the column into a codeword.
template <bool VALUES>
__device__ int decode_column(const LocateTables& t, const u8* s, int k, int m, int radius, int* a, int* b, u8* ea, u8* eb) {
    u8 L[SWEC_MAX_SHARDS];
    u32 nz = 0;
    for (int i = 0; i < m; i++) {
        L[i] = t.log[s[i]];
        if (s[i]) nz |= 1u << i;
    }
    const int w = __popc(nz);
    if (w == 1) {
        *a = k + __ffs(nz) - 1;
        if (VALUES) *ea = s[*a - k];
        return 1;
    }
    if (w == m)  // every entry of an MDS P is non-zero
        for (int j = 0; j < k; j++) {
            int r;
            if (multiple_of_column(t, L, m, j, -1, r)) {
                *a = j;
                if (VALUES) *ea = t.exp[r];
                return 1;
            }
        }
    if (radius < 2) return 0;
    if (w == 2) {
        *a = k + __ffs(nz) - 1;
        *b = k + __ffs(nz & (nz - 1)) - 1;
        if (VALUES) {
            *ea = s[*a - k];
            *eb = s[*b - k];
        }
        return 2;
    }
    if (w < m - 1) return 0;  // a data shard in the pattern makes at least m-1 components non-zero
    for (int q = 0; q < m; q++) {
        if (w == m - 1 && ((nz >> q) & 1)) continue;  // the zero component can only be the parity shard's
        for (int j = 0; j < k; j++) {
            int r;
            if (multiple_of_column(t, L, m, j, q, r)) {
                *a = j;
                *b = k + q;
                if (VALUES) {  // s_q = P[q][j]·e_j ^ e_q
                    *ea = t.exp[r];
                    *eb = s[q] ^ t.exp[r + t.logp[q * 32 + j]];
                }
                return 2;
            }
        }
    }
    for (int x = 0; x + 1 < k; x++)
        for (int y = x + 1; y < k; y++) {
            // [P0x P0y; P1x P1y]·[ex; ey] = [s0; s1]
            const u8 nx = gmul(t, t.logp[32 + y], s[0]) ^ gmul(t, t.logp[y], s[1]);
            const u8 ny = gmul(t, t.logp[32 + x], s[0]) ^ gmul(t, t.logp[x], s[1]);
            if (!nx || !ny) continue;
            const int ld = t.logdet[x * 32 + y];
            int lx = int(t.log[nx]) - ld, ly = int(t.log[ny]) - ld;
            if (lx < 0) lx += 255;
            if (ly < 0) ly += 255;
            bool ok = true;
            for (int i = 2; i < m && ok; i++) ok = (t.exp[lx + t.logp[i * 32 + x]] ^ t.exp[ly + t.logp[i * 32 + y]]) == s[i];
            if (ok) {
                *a = x;
                *b = y;
                if (VALUES) {
                    *ea = t.exp[lx];
                    *eb = t.exp[ly];
                }
                return 2;
            }
        }
    return 0;
}

}  // namespace

}  // namespace swec
