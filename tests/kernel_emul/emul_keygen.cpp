// TEST-ONLY serial execution of the permutation-polynomial kernels (keygen.cuh) with the launch shapes of capi_poly.cu.
#include <cstring>
#include <vector>
#include "keygen.cuh"
using namespace h2;

template <class P> static fe load_mont(const uint8_t *b) { fe x; memcpy(x.v, b, 32); return fe_to_mont<P>(x); }
template <class P> static void store_canon(uint8_t *b, const fe &x) { fe r = fe_from_mont<P>(x); memcpy(b, r.v, 32); }

template <class P> static std::vector<fe> tables(const uint8_t *omega, const uint8_t *delta, uint32_t k, uint32_t cols) {
    const uint64_t tlen = KeygenOps<P>::table_len(k, cols);
    std::vector<fe> tab(tlen);
    const fe w = load_mont<P>(omega), d = load_mont<P>(delta);
    const uint64_t threads = (tlen + 127) / 128 * 128;          // the grid capi_poly.cu launches, idle threads included
    for (uint64_t t = 0; t < threads; t++) KeygenOps<P>::tables_body(tab.data(), w, d, k, cols, t);
    return tab;
}
// out: the table [omega^t, t < 2^h | (omega^(2^h))^t, t < 2^(k-h) | delta^c, c < cols] in canonical form; returns its length
extern "C" uint64_t emu_keygen_tables(int field, const uint8_t *omega, const uint8_t *delta, uint32_t k, uint32_t cols, uint8_t *out) {
    if (field == 0) {
        std::vector<fe> tab = tables<FpParams>(omega, delta, k, cols);
        for (size_t t = 0; t < tab.size(); t++) store_canon<FpParams>(out + 32 * t, tab[t]);
        return tab.size();
    }
    std::vector<fe> tab = tables<FqParams>(omega, delta, k, cols);
    for (size_t t = 0; t < tab.size(); t++) store_canon<FqParams>(out + 32 * t, tab[t]);
    return tab.size();
}
extern "C" uint32_t emu_keygen_split(uint32_t k) { return KeygenOps<FpParams>::split(k); }

// dst: cols * 2^k canonical elements, column after column; mapping: cols * 2^k (column, row) pairs.  The pieces and the
// error word of capi_poly.cu's permutation_sigma_run (piece = rows per launch); returns the error word.
template <class P>
static int run_sigma(const uint32_t *mapping, uint32_t cols, uint32_t k, const uint8_t *omega, const uint8_t *delta, uint64_t piece, uint8_t *dst) {
    const uint64_t n = 1ull << k;
    std::vector<fe> tab = tables<P>(omega, delta, k, cols), col(n);
    uint32_t err = 0;
    for (uint64_t i = 0; i < cols; i++) {
        for (uint64_t j = 0; j < n; j++) col[j] = load_mont<P>(dst + 32 * (i * n + j));
        for (uint64_t j0 = 0; j0 < n; j0 += piece) {
            const uint64_t len = n - j0 < piece ? n - j0 : piece;
            const uint2 *map = reinterpret_cast<const uint2 *>(mapping + 2 * (i * n + j0));
            const uint64_t threads = (len + 255) / 256 * 256;
            for (uint64_t t = 0; t < threads; t++)
                if (KeygenOps<P>::sigma_body(col.data() + j0, map, tab.data(), k, cols, len, t)) err = 1;
        }
        for (uint64_t j = 0; j < n; j++) store_canon<P>(dst + 32 * (i * n + j), col[j]);
    }
    return (int)err;
}
extern "C" int emu_permutation_sigma(int field, const uint32_t *mapping, uint32_t cols, uint32_t k, const uint8_t *omega, const uint8_t *delta,
                                     uint64_t piece, uint8_t *dst_io) {
    return field == 0 ? run_sigma<FpParams>(mapping, cols, k, omega, delta, piece, dst_io)
                      : run_sigma<FqParams>(mapping, cols, k, omega, delta, piece, dst_io);
}
