// TEST-ONLY serial execution of the product-column kernels (grandproduct.cuh) with the launch schedule of capi_poly.cu's
// product_run: power tables, factors, batch inversion over the flat scratch, the batched chunk tree, carries, blinding rows.
#include <cstring>
#include <vector>
#include "grandproduct.cuh"
using namespace h2;

template <class P> static fe load_mont(const uint8_t *b) { fe x; memcpy(x.v, b, 32); return fe_to_mont<P>(x); }
template <class P> static void store_canon(uint8_t *b, const fe &x) { fe r = fe_from_mont<P>(x); memcpy(b, r.v, 32); }
static uint64_t grid(uint64_t n, uint64_t bs) { return (n + bs - 1) / bs * bs; }   // threads of a launch, idle ones included

// perm: ins = proofs x ncols columns then ncols sigmas (n canonical elements each); lookup: 4 per column.  z_out: count x n.
template <class P>
static void run(bool perm, const uint8_t *ins_in, uint64_t n_ins, uint32_t ncols, uint32_t chunk_len, uint32_t sets, uint64_t count, uint32_t k,
                const uint8_t *beta, const uint8_t *gamma, const uint8_t *omega, const uint8_t *delta, const uint8_t *blinding, uint32_t bf,
                uint8_t *z_out) {
    const uint64_t n = 1ull << k;
    std::vector<std::vector<fe>> ins(n_ins, std::vector<fe>(n)), z(count, std::vector<fe>(n));
    std::vector<const fe *> ip(n_ins);
    std::vector<fe *> zp(count);
    for (uint64_t c = 0; c < n_ins; c++) {
        for (uint64_t i = 0; i < n; i++) ins[c][i] = load_mont<P>(ins_in + 32 * (c * n + i));
        ip[c] = ins[c].data();
    }
    for (uint64_t b = 0; b < count; b++) zp[b] = z[b].data();
    GpLevels G{};
    G.m[0] = n; G.m[1] = (n + H2_POLY_CHUNK - 1) / H2_POLY_CHUNK; G.L = 1;
    while (G.m[G.L] > H2_POLY_CHUNK) { G.off[G.L + 1] = G.off[G.L] + G.m[G.L] * count; G.m[G.L + 1] = (G.m[G.L] + H2_POLY_CHUNK - 1) / H2_POLY_CHUNK; G.L++; }
    const uint64_t total = G.off[G.L] + G.m[G.L] * count;
    std::vector<fe> val(count * n), lvl(total), ex(total), init(count), blind(count * bf);
    for (uint64_t j = 0; j < count * bf; j++) blind[j] = load_mont<P>(blinding + 32 * j);
    const fe b_m = load_mont<P>(beta), g_m = load_mont<P>(gamma);
    if (perm) {
        const uint64_t tlen = KeygenOps<P>::table_len(k, ncols);
        std::vector<fe> tab(tlen);
        for (uint64_t t = 0; t < grid(tlen, 128); t++) KeygenOps<P>::tables_body(tab.data(), load_mont<P>(omega), load_mont<P>(delta), k, ncols, t);
        for (uint32_t b = 0; b < count; b++)
            for (uint64_t i = 0; i < grid(n, 128); i++)
                ProductArgs<P>::perm_factors_body(ip.data(), ip.data() + (count / sets) * ncols, ncols, chunk_len, sets, tab.data(), k, b_m, g_m,
                                                  val.data(), zp.data(), b, i);
    } else {
        for (uint32_t b = 0; b < count; b++)
            for (uint64_t i = 0; i < grid(n, 256); i++) ProductArgs<P>::lookup_factors_body(ip.data(), n, b_m, g_m, val.data(), zp.data(), b, i);
    }
    for (uint64_t t = 0; t < grid((count * n + 15) / 16, 64); t++) GrandProduct<P>::invert_body(val.data(), count * n, t);
    for (uint32_t b = 0; b < count; b++)
        for (uint64_t t = 0; t < grid(G.m[1], 128); t++) ProductArgs<P>::mv_up_body(zp.data(), val.data(), n, lvl.data(), G.m[1], b, t);
    for (uint32_t l = 1; l < G.L; l++)
        for (uint64_t b = 0; b < count; b++)
            for (uint64_t t = 0; t < grid(G.m[l + 1], 128); t++)
                GrandProduct<P>::up_body(lvl.data() + G.off[l] + b * G.m[l], G.m[l], lvl.data() + G.off[l + 1] + b * G.m[l + 1], G.m[l + 1], t);
    for (uint32_t p = 0; p < count / sets; p++) ProductArgs<P>::carry_body(val.data(), lvl.data(), G, n - bf - 1, sets, init.data(), p);
    for (uint32_t l = G.L + 1; l-- > 0;) {
        const uint64_t chunks = (G.m[l] + H2_POLY_CHUNK - 1) / H2_POLY_CHUNK;
        for (uint64_t b = 0; b < count; b++)
            for (uint64_t t = 0; t < grid(chunks, 128); t++)
                GrandProduct<P>::down_body(l == 0 ? val.data() + b * n : lvl.data() + G.off[l] + b * G.m[l], G.m[l],
                                           l == G.L ? nullptr : ex.data() + G.off[l + 1] + b * chunks, init[b],
                                           l == 0 ? zp[b] : ex.data() + G.off[l] + b * G.m[l], chunks, t);
    }
    for (uint64_t j = 0; j < grid(count * bf, 256); j++) ProductArgs<P>::blind_body(zp.data(), n, bf, blind.data(), count, j);
    for (uint64_t b = 0; b < count; b++)
        for (uint64_t i = 0; i < n; i++) store_canon<P>(z_out + 32 * (b * n + i), z[b][i]);
}

extern "C" void emu_permutation_product(int field, const uint8_t *columns_then_sigmas, uint32_t proofs, uint32_t cols, uint32_t chunk_len, uint32_t k,
                                        const uint8_t *beta, const uint8_t *gamma, const uint8_t *omega, const uint8_t *delta, const uint8_t *blinding,
                                        uint32_t bf, uint8_t *z_out) {
    const uint32_t sets = (cols + chunk_len - 1) / chunk_len;
    auto f = field == 0 ? run<FpParams> : run<FqParams>;
    f(true, columns_then_sigmas, (uint64_t)(proofs + 1) * cols, cols, chunk_len, sets, (uint64_t)proofs * sets, k, beta, gamma, omega, delta, blinding, bf,
      z_out);
}
extern "C" void emu_lookup_product(int field, const uint8_t *io, uint32_t count, uint32_t k, const uint8_t *beta, const uint8_t *gamma,
                                   const uint8_t *blinding, uint32_t bf, uint8_t *z_out) {
    auto f = field == 0 ? run<FpParams> : run<FqParams>;
    f(false, io, 4ull * count, 0, 1, 1, count, k, beta, gamma, nullptr, nullptr, blinding, bf, z_out);
}
