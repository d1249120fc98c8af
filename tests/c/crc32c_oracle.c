/* tests/c/crc32c_oracle.c — the host CRC32-C (Castagnoli) the needle-check tests and benchmark compare against.
 * Checker only: SSE4.2 crc32 instructions where the CPU has them, a byte table otherwise.  Besides the plain update it
 * gives, over many threads, the CRC of byte ranges of memory, and of byte ranges of the seeded synthetic stream
 * (swec_synth_fill_device: byte b = byte b%8 of splitmix64(seed + (b/8 + 1)·0x9E3779B97F4A7C15)) without ever
 * holding the stream in memory. */
#include <pthread.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

static uint32_t table[256];
static int have_hw = -1;

static void init(void) {
    if (have_hw >= 0) return;
    for (uint32_t i = 0; i < 256; i++) {
        uint32_t c = i;
        for (int b = 0; b < 8; b++) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
        table[i] = c;
    }
#if defined(__x86_64__)
    __builtin_cpu_init();
    have_hw = __builtin_cpu_supports("sse4.2") ? 1 : 0;
#else
    have_hw = 0;
#endif
}

static uint32_t update_sw(uint32_t c, const uint8_t *p, size_t n) {
    while (n--) c = table[(c ^ *p++) & 0xffu] ^ (c >> 8);
    return c;
}

#if defined(__x86_64__)
__attribute__((target("sse4.2"))) static uint32_t update_hw(uint32_t c, const uint8_t *p, size_t n) {
    uint64_t c64 = c;
    while (n >= 8) {
        uint64_t w;
        memcpy(&w, p, 8);
        c64 = __builtin_ia32_crc32di(c64, w);
        p += 8;
        n -= 8;
    }
    c = (uint32_t)c64;
    while (n--) c = __builtin_ia32_crc32qi(c, *p++);
    return c;
}
#endif

/* Go's crc32.Update(crc, crc32.MakeTable(crc32.Castagnoli), p[:n]) */
uint32_t orc_crc32c_update(uint32_t crc, const uint8_t *p, size_t n) {
    init();
    uint32_t c = ~crc;
#if defined(__x86_64__)
    if (have_hw) return ~update_hw(c, p, n);
#endif
    return ~update_sw(c, p, n);
}

int orc_crc32c_has_hw(void) {
    init();
    return have_hw;
}

static uint64_t splitmix64_at(uint64_t seed, uint64_t j) {
    uint64_t z = seed + (j + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

struct job {
    const uint8_t *base; /* NULL: the synthetic stream */
    uint64_t seed;
    const int64_t *off, *len;
    uint32_t *out;
    int n;
    int next; /* shared cursor */
};

static void *worker(void *arg) {
    struct job *j = arg;
    uint8_t buf[1 << 16];
    for (;;) {
        const int r = __atomic_fetch_add(&j->next, 1, __ATOMIC_RELAXED);
        if (r >= j->n) break;
        uint32_t crc = 0;
        if (j->base) {
            crc = orc_crc32c_update(0, j->base + j->off[r], (size_t)j->len[r]);
        } else {
            int64_t at = j->off[r], left = j->len[r];
            while (left > 0) {
                /* whole words of the stream covering [at, at + piece) */
                const int64_t piece = left < (int64_t)sizeof buf - 16 ? left : (int64_t)sizeof buf - 16;
                const uint64_t w0 = (uint64_t)at / 8, w1 = ((uint64_t)(at + piece) + 7) / 8;
                uint8_t *q = buf;
                for (uint64_t w = w0; w < w1; w++, q += 8) {
                    const uint64_t v = splitmix64_at(j->seed, w);
                    memcpy(q, &v, 8); /* little-endian hosts */
                }
                crc = orc_crc32c_update(crc, buf + (at - (int64_t)w0 * 8), (size_t)piece);
                at += piece;
                left -= piece;
            }
        }
        j->out[r] = crc;
    }
    return NULL;
}

static int run(struct job *j, int threads) {
    init();
    if (threads < 1) threads = 1;
    if (threads > 256) threads = 256;
    pthread_t t[256];
    int started = 0;
    for (; started < threads - 1; started++)
        if (pthread_create(&t[started], NULL, worker, j) != 0) break;
    worker(j);
    for (int i = 0; i < started; i++) pthread_join(t[i], NULL);
    return 0;
}

/* out[r] = CRC32-C of base[off[r], off[r] + len[r]) */
int orc_crc32c_ranges(const uint8_t *base, const int64_t *off, const int64_t *len, uint32_t *out, int n, int threads) {
    struct job j = {base, 0, off, len, out, n, 0};
    return run(&j, threads);
}

/* out[r] = CRC32-C of bytes [off[r], off[r] + len[r]) of the synthetic stream of `seed` */
int orc_synth_crc32c(uint64_t seed, const int64_t *off, const int64_t *len, uint32_t *out, int n, int threads) {
    struct job j = {NULL, seed, off, len, out, n, 0};
    return run(&j, threads);
}
