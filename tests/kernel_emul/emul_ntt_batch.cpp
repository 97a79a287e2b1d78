// TEST-ONLY serial execution of the column-batched NTT passes (ntt.cuh; the pass loop of capi_ntt.cu's ntt_run) on the host:
// `count` columns of one size and domain, column c = blockIdx.y of every launch, each column in its own allocation reached
// through the in_cols / out_cols tables, the intermediate passes in one scratch slot per column of a group.
#include <cstring>
#include <vector>
#include "ntt.cuh"
using namespace h2;

// mode 1: ifft (out_scale = divisor); 2: coeff_to_extended (in_log_n = k, in_scale zeta powers).  Elements canonical, column
// by column: in holds count x 2^in_log_n, out count x 2^log_n.  group: columns per launch (0 = ntt_group's plan); in_place:
// out_cols[c] == in_cols[c] (needs in_log_n == log_n).  Returns the number of launches.
template <class P>
static int run_batch(int mode, const uint8_t *in, uint64_t count, uint32_t in_log_n, uint32_t log_n, const uint8_t *omega, const uint8_t *zeta,
                     const uint8_t *divisor, uint8_t *out, uint64_t group, int in_place, uint32_t nthr) {
    const uint64_t n = 1ull << log_n, n_in = 1ull << in_log_n;
    std::vector<std::vector<fe>> src(count, std::vector<fe>(n)), dst(count, std::vector<fe>(n));
    for (uint64_t c = 0; c < count; c++)
        for (uint64_t i = 0; i < n_in; i++) memcpy(src[c][i].v, in + 32 * (c * n_in + i), 32);
    std::vector<const fe *> in_cols(count);
    std::vector<fe *> out_cols(count);
    for (uint64_t c = 0; c < count; c++) { in_cols[c] = src[c].data(); out_cols[c] = in_place ? src[c].data() : dst[c].data(); }
    fe w, z = fe_zero(), dv = fe_zero();
    memcpy(w.v, omega, 32); w = fe_to_mont<P>(w);
    if (zeta) { memcpy(z.v, zeta, 32); z = fe_to_mont<P>(z); }
    if (divisor) { memcpy(dv.v, divisor, 32); dv = fe_to_mont<P>(dv); }
    std::vector<fe> tw(n / 2 ? n / 2 : 1), pow2(32);
    TwiddleGen<P>::pow2_body(pow2.data(), w, log_n ? log_n : 1);
    for (uint64_t t = 0; t * 32 < (n / 2); t++) TwiddleGen<P>::fill_body(tw.data(), pow2.data(), n / 2, t);
    uint32_t sp[8], logc[8];
    int passes = ntt_plan(log_n, sp, logc);
    if (passes == 0) { sp[0] = 0; logc[0] = 0; passes = 1; }
    if (group == 0) group = ntt_group(log_n, passes, count);
    std::vector<fe> work(passes > 1 ? group * n : 1);
    // canonical in / out folded into the scales, as emul_ntt.cpp does
    const fe zp[3] = {fe_one<P>(), z, fe_mul<P>(z, z)};
    fe one_c = fe_zero(); one_c.v[0] = 1;
    int launches = 0;
    for (uint64_t c0 = 0; c0 < count; c0 += group) {
        const uint32_t cols = (uint32_t)(count - c0 < group ? count - c0 : group);
        uint32_t s0 = 0;
        for (int i = 0; i < passes; i++) {
            NttPassArgs A;
            A.in = i == 0 ? nullptr : work.data();
            A.out = i == passes - 1 ? nullptr : work.data();
            if (i > 0) A.in_stride = n;
            if (i < passes - 1) A.out_stride = n;
            if (i == 0) A.in_cols = in_cols.data() + c0;
            if (i == passes - 1) A.out_cols = out_cols.data() + c0;
            A.tw = tw.data(); A.log_n = log_n; A.s0 = s0; A.sp = sp[i]; A.logc = logc[i];
            A.flags = (i == 0 ? NTT_FIRST | NTT_IN_SCALE : 0) | (i == passes - 1 ? NTT_LAST | NTT_OUT_SCALE : 0);
            A.in_log_n = in_log_n; A.out_len = n;
            for (int k = 0; k < 3; k++) A.in_scale[k] = mode == 2 ? fe_mul<P>(zp[k], fe_r2<P>()) : fe_r2<P>();
            for (int k = 0; k < 3; k++) A.out_scale[k] = mode == 1 ? fe_from_mont<P>(dv) : one_c;
            const uint32_t tiles = (uint32_t)(n >> (sp[i] + logc[i]));
            std::vector<uint4> sm(ntt_smem_bytes(sp[i], logc[i]) / 16), twc(ntt_twc_bytes(sp[i], logc[i], i == passes - 1) / 16 + 1);
            launches++;
            // one launch: grid (tiles, cols), the phase order of ntt_pass_kernel.  Blocks of one launch may run in any order;
            // visiting the columns last-first shows that no column depends on another.
            for (uint32_t y = cols; y-- > 0;)
                for (uint32_t tile = 0; tile < tiles; tile++) {
                    for (uint32_t t = 0; t < nthr; t++) NttPass<P>::twiddle_phase(A, tile, t, nthr, twc.data());
                    for (uint32_t t = 0; t < nthr; t++) NttPass<P>::load_phase(A, tile, t, nthr, sm.data(), y);
                    for (uint32_t st = 0; st < NttPass<P>::num_steps(sp[i]); st++)
                        for (uint32_t t = 0; t < nthr; t++) NttPass<P>::step_phase(A, tile, st, t, nthr, sm.data(), twc.data());
                    for (uint32_t t = 0; t < nthr; t++) NttPass<P>::store_phase(A, tile, t, nthr, sm.data(), y);
                }
            s0 += sp[i];
        }
    }
    for (uint64_t c = 0; c < count; c++)
        for (uint64_t i = 0; i < n; i++) memcpy(out + 32 * (c * n + i), out_cols[c][i].v, 32);
    return launches;
}
extern "C" int emu_ntt_batch(int field, int mode, const uint8_t *in, uint64_t count, uint32_t in_log_n, uint32_t log_n, const uint8_t *omega,
                             const uint8_t *zeta, const uint8_t *divisor, uint8_t *out, uint64_t group, int in_place, uint32_t nthr) {
    if (field == 0) return run_batch<FpParams>(mode, in, count, in_log_n, log_n, omega, zeta, divisor, out, group, in_place, nthr);
    return run_batch<FqParams>(mode, in, count, in_log_n, log_n, omega, zeta, divisor, out, group, in_place, nthr);
}
