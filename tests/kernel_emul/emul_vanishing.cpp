// TEST-ONLY serial execution of h2_poly_vanishing_quotient's pass loop (capi_ntt.cu; ntt.cuh, NTT_IN_TABLE / NTT_OUT_PIECES)
// on the host: one extended-domain column, the division by t(X) on the first pass's loads, the inverse transform, the zeta
// un-shift and 1 / 2^ext_k on the last pass's stores, which scatter the coefficients into `count` pieces of 2^k, each in its
// own allocation reached through the piece table.
#include <cstring>
#include <vector>
#include "ntt.cuh"
using namespace h2;

// src: 2^ext_k canonical elements; out: count x 2^k canonical elements, piece by piece.  reverse: every launch visits its
// tiles last-first.  Returns the number of launches, -1 when vanishing_quotient_sizes rejects the sizes, -2 when a store
// landed outside [0, 2^k) of its piece.
template <class P>
static int run(const uint8_t *src, uint32_t k, uint32_t ext_k, uint64_t count, const uint8_t *omega_inv, const uint8_t *divisor,
               const uint8_t *zeta, const uint8_t *t_evals, uint32_t t_len, uint8_t *out, int reverse, uint32_t nthr) {
    if (vanishing_quotient_sizes(k, ext_k, count, t_len)) return -1;
    const uint64_t n = 1ull << k, N = 1ull << ext_k;
    auto mont = [](const uint8_t *b) { fe x; memcpy(x.v, b, 32); return fe_to_mont<P>(x); };
    std::vector<fe> in(N), table(t_len);
    for (uint64_t i = 0; i < N; i++) in[i] = mont(src + 32 * i);
    for (uint32_t i = 0; i < t_len; i++) table[i] = mont(t_evals + 32 * i);
    // one guard element after every piece: the last pass must not write past 2^k
    fe guard;
    for (int w = 0; w < 8; w++) guard.v[w] = 0xA5A5A5A5u;
    std::vector<std::vector<fe>> pieces(count, std::vector<fe>(n + 1, guard));
    std::vector<fe *> cols(count);
    for (uint64_t c = 0; c < count; c++) cols[c] = pieces[c].data();
    const fe w = mont(omega_inv), d = mont(divisor), z = mont(zeta);
    std::vector<fe> tw(N / 2 ? N / 2 : 1), pow2(32);
    TwiddleGen<P>::pow2_body(pow2.data(), w, ext_k ? ext_k : 1);
    for (uint64_t t = 0; t * 32 < (N / 2); t++) TwiddleGen<P>::fill_body(tw.data(), pow2.data(), N / 2, t);
    uint32_t sp[8], logc[8];
    int passes = ntt_plan(ext_k, sp, logc);
    if (passes == 0) { sp[0] = 0; logc[0] = 0; passes = 1; }
    std::vector<fe> work(passes > 1 ? N : 1);
    // make_scales(canon = false, divisor, zeta_out): [d, d zeta^2, d zeta] on output p mod 3
    const fe out_s[3] = {d, fe_mul<P>(d, fe_mul<P>(z, z)), fe_mul<P>(d, z)};
    uint32_t s0 = 0;
    for (int i = 0; i < passes; i++) {
        NttPassArgs A;
        A.in = i == 0 ? in.data() : work.data();
        A.out = i == passes - 1 ? nullptr : work.data();
        if (i == passes - 1) A.out_cols = cols.data();
        A.tw = tw.data(); A.log_n = ext_k; A.s0 = s0; A.sp = sp[i]; A.logc = logc[i];
        A.flags = (i == 0 ? NTT_FIRST | NTT_IN_TABLE : 0) | (i == passes - 1 ? NTT_LAST | NTT_OUT_SCALE | NTT_OUT_PIECES : 0);
        A.in_log_n = ext_k; A.out_len = count << k;
        A.in_table = table.data(); A.in_mask = t_len - 1; A.piece_log = k;
        for (int j = 0; j < 3; j++) A.out_scale[j] = out_s[j];
        const uint32_t tiles = (uint32_t)(N >> (sp[i] + logc[i]));
        std::vector<uint4> sm(ntt_smem_bytes(sp[i], logc[i]) / 16), twc(ntt_twc_bytes(sp[i], logc[i], i == passes - 1) / 16 + 1);
        for (uint32_t b = 0; b < tiles; b++) {
            const uint32_t tile = reverse ? tiles - 1 - b : b;
            for (uint32_t t = 0; t < nthr; t++) NttPass<P>::twiddle_phase(A, tile, t, nthr, twc.data());
            for (uint32_t t = 0; t < nthr; t++) NttPass<P>::load_phase(A, tile, t, nthr, sm.data());
            for (uint32_t st = 0; st < NttPass<P>::num_steps(sp[i]); st++)
                for (uint32_t t = 0; t < nthr; t++) NttPass<P>::step_phase(A, tile, st, t, nthr, sm.data(), twc.data());
            for (uint32_t t = 0; t < nthr; t++) NttPass<P>::store_phase(A, tile, t, nthr, sm.data());
        }
        s0 += sp[i];
    }
    for (uint64_t c = 0; c < count; c++) {
        if (memcmp(pieces[c][n].v, guard.v, 32)) return -2;
        for (uint64_t i = 0; i < n; i++) {
            const fe x = fe_from_mont<P>(pieces[c][i]);
            memcpy(out + 32 * (c * n + i), x.v, 32);
        }
    }
    return passes;
}
extern "C" int emu_vanishing_quotient(int field, const uint8_t *src, uint32_t k, uint32_t ext_k, uint64_t count, const uint8_t *omega_inv,
                                      const uint8_t *divisor, const uint8_t *zeta, const uint8_t *t_evals, uint32_t t_len, uint8_t *out,
                                      int reverse, uint32_t nthr) {
    if (field == 0) return run<FpParams>(src, k, ext_k, count, omega_inv, divisor, zeta, t_evals, t_len, out, reverse, nthr);
    return run<FqParams>(src, k, ext_k, count, omega_inv, divisor, zeta, t_evals, t_len, out, reverse, nthr);
}
// the reason vanishing_quotient_sizes gives, or nullptr
extern "C" const char *emu_vanishing_quotient_sizes(uint32_t k, uint32_t ext_k, uint64_t count, uint32_t t_len) {
    return vanishing_quotient_sizes(k, ext_k, count, t_len);
}
