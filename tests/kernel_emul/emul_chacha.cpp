// TEST-ONLY serial execution of K26 (chacha.cuh): the keystream block, the 512-bit reduction, and h2_poly_random's kernel
// over its whole grid.
#include <cstring>
#include <vector>
#include "chacha.cuh"
using namespace h2;

static ChaChaKey key_of(const uint8_t *seed) {
    ChaChaKey k;
    memcpy(k.k, seed, sizeof k.k);
    return k;
}

// out: the 16 words of keystream block `block`
extern "C" void emu_chacha_block(const uint8_t *seed, uint64_t stream, uint64_t block, uint32_t *out) {
    uint32_t w[16];
    chacha_block(key_of(seed), stream, block, w);
    memcpy(out, w, sizeof w);
}

// n 64-byte little-endian integers -> their residues mod m, canonical 32 bytes each (from_u512, then out of Montgomery form)
template <class P> static void run_reduce(const uint8_t *in, uint64_t n, uint8_t *out) {
    for (uint64_t i = 0; i < n; i++) {
        uint32_t w[16];
        memcpy(w, in + 64 * i, 64);
        const fe r = fe_from_mont<P>(ChaChaRandom<P>::from_u512(w));
        memcpy(out + 32 * i, r.v, 32);
    }
}
extern "C" void emu_chacha_reduce(int field, const uint8_t *in, uint64_t n, uint8_t *out) {
    field == 0 ? run_reduce<FpParams>(in, n, out) : run_reduce<FqParams>(in, n, out);
}

// h2_poly_random's launch: `count` polynomials of lens[i] elements, every (polynomial, element) of the grid through the kernel
// body in Montgomery form; out: the polynomials one after another, canonical.
template <class P>
static void run_random(const uint8_t *seed, uint64_t stream, uint64_t block, uint32_t word, uint64_t count, const uint64_t *lens, uint8_t *out) {
    const ChaChaKey key = key_of(seed);
    std::vector<RandCol> cols(count);
    uint64_t total = 0, longest = 0;
    for (uint64_t c = 0; c < count; c++) {
        cols[c] = {total, lens[c]};
        total += lens[c];
        if (lens[c] > longest) longest = lens[c];
    }
    std::vector<fe> res(total);
    for (uint64_t c = 0; c < count; c++)
        for (uint64_t i = 0; i < longest; i++) ChaChaRandom<P>::body(res.data() + cols[c].first, cols[c], key, stream, block, word, i);
    for (uint64_t j = 0; j < total; j++) {
        const fe r = fe_from_mont<P>(res[j]);
        memcpy(out + 32 * j, r.v, 32);
    }
}
extern "C" void emu_chacha_random(int field, const uint8_t *seed, uint64_t stream, uint64_t block, uint32_t word, uint64_t count, const uint64_t *lens,
                                  uint8_t *out) {
    field == 0 ? run_random<FpParams>(seed, stream, block, word, count, lens, out) : run_random<FqParams>(seed, stream, block, word, count, lens, out);
}
