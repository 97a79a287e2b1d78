/* The draws of a seeded rand_chacha 0.3.1 ChaCha20Rng through pasta_curves 0.5.1's Field::random, in C (TEST
 * INFRASTRUCTURE ONLY -- see pasta.py): the oracle of the device draws (csrc/chacha.cuh, K26) at GPU sizes, and the timed
 * single-thread CPU baseline of tools/random_poly_time.py.
 *
 * Keystream: RFC 8439 section 2.3's block function over bytes, key = the seed, state words 12-13 a 64-bit block counter and
 * words 14-15 a 64-bit stream id (rand_chacha's layout); the words are read in order, little-endian.
 * Field::random: from_u512 of eight next_u64, i.e. the 64 bytes as one little-endian 512-bit integer, mod m.  The residue is
 * taken here by long division, 32 bits at a time with the quotient estimated from the top bits (m = 2^254 + t, t < 2^126),
 * not by the device's Montgomery products. */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

typedef unsigned __int128 u128;

static const uint64_t MODULI[2][4] = {
    {0x992d30ed00000001ull, 0x224698fc094cf91bull, 0x0ull, 0x4000000000000000ull},   /* fp */
    {0x8c46eb2100000001ull, 0x224698fc0994a8ddull, 0x0ull, 0x4000000000000000ull},   /* fq */
};

static uint32_t ld32(const uint8_t *p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
static uint32_t rotl(uint32_t x, int n) { return (x << n) | (x >> (32 - n)); }

#define QR(a, b, c, d)                                  \
    do {                                                \
        a += b; d ^= a; d = rotl(d, 16);                \
        c += d; b ^= c; b = rotl(b, 12);                \
        a += b; d ^= a; d = rotl(d, 8);                 \
        c += d; b ^= c; b = rotl(b, 7);                 \
    } while (0)

static void block_words(const uint8_t key[32], uint64_t stream, uint64_t counter, uint32_t out[16]) {
    static const uint8_t sigma[16] = "expand 32-byte k";
    uint32_t s[16], x[16];
    for (int i = 0; i < 4; i++) s[i] = ld32(sigma + 4 * i);
    for (int i = 0; i < 8; i++) s[4 + i] = ld32(key + 4 * i);
    s[12] = (uint32_t)counter;
    s[13] = (uint32_t)(counter >> 32);
    s[14] = (uint32_t)stream;
    s[15] = (uint32_t)(stream >> 32);
    memcpy(x, s, sizeof x);
    for (int r = 0; r < 10; r++) {
        QR(x[0], x[4], x[8], x[12]); QR(x[1], x[5], x[9], x[13]); QR(x[2], x[6], x[10], x[14]); QR(x[3], x[7], x[11], x[15]);
        QR(x[0], x[5], x[10], x[15]); QR(x[1], x[6], x[11], x[12]); QR(x[2], x[7], x[8], x[13]); QR(x[3], x[4], x[9], x[14]);
    }
    for (int i = 0; i < 16; i++) out[i] = x[i] + s[i];
}

/* nwords keystream words from word position 16 * block + word (word < 16) */
int orc_chacha_words(const uint8_t *key, uint64_t stream, uint64_t block, uint32_t word, uint64_t nwords, uint32_t *out) {
    if (word >= 16) return 1;
    uint32_t b[16];
    block_words(key, stream, block, b);
    for (uint64_t i = 0; i < nwords; i++) {
        if (word == 16) { block_words(key, stream, ++block, b); word = 0; }
        out[i] = b[word++];
    }
    return 0;
}

/* r = (r 2^32 + w) mod m for r < m */
static void shift_in(const uint64_t m[4], uint64_t r[4], uint32_t w) {
    uint64_t t[5];
    t[0] = (r[0] << 32) | w;
    t[1] = (r[1] << 32) | (r[0] >> 32);
    t[2] = (r[2] << 32) | (r[1] >> 32);
    t[3] = (r[3] << 32) | (r[2] >> 32);
    t[4] = r[3] >> 32;
    /* q = floor(t / 2^254) is floor(t / m) or one more: t < m 2^32, so t / 2^254 - t / m = t (m - 2^254) / (2^254 m) < 2^-96 */
    const uint64_t q = (t[3] >> 62) | (t[4] << 2);
    uint64_t borrow = 0, carry = 0;
    for (int i = 0; i < 5; i++) {
        const u128 p = (u128)q * (i < 4 ? m[i] : 0) + carry;
        carry = (uint64_t)(p >> 64);
        const u128 d = (u128)t[i] - (uint64_t)p - borrow;
        t[i] = (uint64_t)d;
        borrow = (uint64_t)(d >> 64) & 1;
    }
    if (borrow) {   /* t - q m < 0: q was one too many */
        uint64_t c = 0;
        for (int i = 0; i < 5; i++) {
            const u128 s = (u128)t[i] + (i < 4 ? m[i] : 0) + c;
            t[i] = (uint64_t)s;
            c = (uint64_t)(s >> 64);
        }
    }
    memcpy(r, t, 4 * sizeof(uint64_t));
}

/* the 64 bytes of one little-endian 512-bit integer -> its residue mod m, 32 canonical bytes */
static void u512_mod(const uint64_t m[4], const uint8_t in[64], uint8_t out[32]) {
    uint64_t r[4] = {0, 0, 0, 0};
    for (int i = 15; i >= 0; i--) shift_in(m, r, ld32(in + 4 * i));
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 8; j++) out[8 * i + j] = (uint8_t)(r[i] >> (8 * j));
}

int orc_u512_mod(int field, const uint8_t *in, uint64_t n, uint8_t *out) {
    if (field != 0 && field != 1) return 1;
    for (uint64_t i = 0; i < n; i++) u512_mod(MODULI[field], in + 64 * i, out + 32 * i);
    return 0;
}

/* n draws of Field::random from word position 16 * block + word: canonical 32 bytes each.  Single-threaded, the way a
 * prover's own loop draws them. */
int orc_chacha_draws(int field, const uint8_t *key, uint64_t stream, uint64_t block, uint32_t word, uint64_t n, uint8_t *out) {
    if ((field != 0 && field != 1) || word >= 16) return 1;
    uint32_t cur[16], nxt[16] = {0}, w[16];
    uint8_t bytes[64];
    block_words(key, stream, block, cur);
    for (uint64_t j = 0; j < n; j++) {
        if (word) {
            block_words(key, stream, block + j + 1, nxt);
            for (int i = 0; i < 16; i++) w[i] = (uint32_t)i + word < 16 ? cur[i + word] : nxt[i + word - 16];
        } else {
            memcpy(w, cur, sizeof w);
            if (j + 1 < n) block_words(key, stream, block + j + 1, nxt);
        }
        for (int i = 0; i < 16; i++)
            for (int b = 0; b < 4; b++) bytes[4 * i + b] = (uint8_t)(w[i] >> (8 * b));
        u512_mod(MODULI[field], bytes, out + 32 * j);
        memcpy(cur, nxt, sizeof cur);
    }
    return 0;
}
