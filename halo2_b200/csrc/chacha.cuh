// K26: the prover's random polynomials drawn on the device (h2_poly_random): the scalars a ChaCha20Rng seeded with `key`
// gives Field::random, one thread per draw, every polynomial of a call in one launch.
//
// rand_chacha 0.3.1's ChaCha20Rng outputs the ChaCha20 keystream (RFC 8439's block function) with the seed as key, a 64-bit
// block counter in state words 12-13 and a 64-bit stream id in words 14-15; next_u64 reads it word after word,
// little-endian.  pasta_curves 0.5.1's Field::random is from_u512 of eight next_u64: (lo + 2^256 hi) mod m, lo and hi the
// first and second 32 bytes.  So draw j, counted from word position 16 block0 + word, is the 16 keystream words starting
// at 16 (block0 + j) + word, and every draw is independent of every other.  With word != 0 a draw spans two blocks and its
// thread computes both; `word` is uniform across a launch, so the shift that picks the 16 words is a uniform branch over
// compile-time register indices.
//
// The grid covers (polynomial, element): blockIdx.y is the polynomial, the x dimension its elements.  Its buffer comes
// from the call's column table (col_table), its first draw index and length from the RandCol entries behind the
// pointers.  The stored value is the Montgomery form of the canonical scalar: the bytes h2_poly_upload stores for it.
#pragma once
#include "field.cuh"

namespace h2 {

struct ChaChaKey { uint32_t k[8]; };     // the 32-byte seed as eight little-endian words
struct RandCol {                         // one polynomial of a call
    uint64_t first;                      // the draw index of its element 0
    uint64_t len;                        // elements drawn
};

#if defined(__CUDA_ARCH__)
H2_D uint32_t cc_rotl16(uint32_t x) { return __byte_perm(x, 0u, 0x1032u); }
H2_D uint32_t cc_rotl8(uint32_t x) { return __byte_perm(x, 0u, 0x2103u); }
H2_D uint32_t cc_rotl12(uint32_t x) { return __funnelshift_l(x, x, 12); }
H2_D uint32_t cc_rotl7(uint32_t x) { return __funnelshift_l(x, x, 7); }
#else
inline uint32_t cc_rotl16(uint32_t x) { return (x << 16) | (x >> 16); }
inline uint32_t cc_rotl8(uint32_t x) { return (x << 8) | (x >> 24); }
inline uint32_t cc_rotl12(uint32_t x) { return (x << 12) | (x >> 20); }
inline uint32_t cc_rotl7(uint32_t x) { return (x << 7) | (x >> 25); }
#endif

H2_HD void cc_quarter(uint32_t &a, uint32_t &b, uint32_t &c, uint32_t &d) {
    a += b; d ^= a; d = cc_rotl16(d);
    c += d; b ^= c; b = cc_rotl12(b);
    a += b; d ^= a; d = cc_rotl8(d);
    c += d; b ^= c; b = cc_rotl7(b);
}

// One 64-byte keystream block as 16 little-endian words (RFC 8439 section 2.3, with rand_chacha's 64-bit counter and
// stream words).
H2_HD void chacha_block(const ChaChaKey &key, uint64_t stream, uint64_t block, uint32_t (&out)[16]) {
    uint32_t x[16];
    x[0] = 0x61707865u; x[1] = 0x3320646eu; x[2] = 0x79622d32u; x[3] = 0x6b206574u;   // "expand 32-byte k"
    for (int i = 0; i < 8; i++) x[4 + i] = key.k[i];
    x[12] = (uint32_t)block; x[13] = (uint32_t)(block >> 32);
    x[14] = (uint32_t)stream; x[15] = (uint32_t)(stream >> 32);
    for (int i = 0; i < 16; i++) out[i] = x[i];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int r = 0; r < 10; r++) {
        cc_quarter(x[0], x[4], x[8], x[12]);
        cc_quarter(x[1], x[5], x[9], x[13]);
        cc_quarter(x[2], x[6], x[10], x[14]);
        cc_quarter(x[3], x[7], x[11], x[15]);
        cc_quarter(x[0], x[5], x[10], x[15]);
        cc_quarter(x[1], x[6], x[11], x[12]);
        cc_quarter(x[2], x[7], x[8], x[13]);
        cc_quarter(x[3], x[4], x[9], x[14]);
    }
    for (int i = 0; i < 16; i++) out[i] += x[i];
}

template <class P> struct ChaChaRandom {
    // The Montgomery form of (lo + 2^256 hi) mod m for the 512-bit integer w[0..16) (little-endian words): from_u512's
    // lo R^2 + hi R^3 through fe_mul.  fe_mul takes operands in [0, m) and a 256-bit half is < 2^256 < 4m, so each half
    // first loses m up to three times.
    static H2_HD fe from_u512(const uint32_t (&w)[16]) {
        fe lo, hi, r3, a, b;
        for (int i = 0; i < 8; i++) { lo.v[i] = w[i]; hi.v[i] = w[8 + i]; r3.v[i] = P::r3(i); }
        for (int t = 0; t < 3; t++) { fe_cond_sub_mod<P>(lo); fe_cond_sub_mod<P>(hi); }
        fe_mul2<P>(a, lo, fe_r2<P>(), b, hi, r3);
        return fe_add<P>(a, b);
    }
    // Draw j from word position 16 block0 + word (word < 16): keystream words 16 (block0 + j) + word ... + 15.
    static H2_HD fe draw(const ChaChaKey &key, uint64_t stream, uint64_t block0, uint32_t word, uint64_t j) {
        uint32_t w[16];
        chacha_block(key, stream, block0 + j, w);
        if (word) {
            uint32_t nx[16];
            chacha_block(key, stream, block0 + j + 1, nx);
            // w ++ nx shifted down by word = 8 b3 + 4 b2 + 2 b1 + b0 words, one shift per set bit
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
            for (uint32_t s = 8; s; s >>= 1) {
                if (word & s) {
                    for (uint32_t i = 0; i < 16; i++) w[i] = i + s < 16 ? w[i + s] : nx[i + s - 16];
                    for (uint32_t i = 0; i + s < 16; i++) nx[i] = nx[i + s];
                }
            }
        }
        return from_u512(w);
    }
    static H2_HD void body(fe *out, const RandCol &c, const ChaChaKey &key, uint64_t stream, uint64_t block0, uint32_t word, uint64_t i) {
        if (i >= c.len) return;
        fe_store(out + i, draw(key, stream, block0, word, c.first + i));
    }
};

#if defined(__CUDACC__)
// polynomials [col0, col0 + gridDim.y) of the table; grid.x covers the longest of them
template <class P>
__global__ void __launch_bounds__(256) chacha_random_kernel(fe *const *polys, const RandCol *cols, uint32_t col0, ChaChaKey key, uint64_t stream,
                                                            uint64_t block0, uint32_t word) {
    const uint32_t c = col0 + blockIdx.y;
    ChaChaRandom<P>::body(polys[c], cols[c], key, stream, block0, word, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
#endif

}  // namespace h2
