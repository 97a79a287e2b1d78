// TEST-ONLY serial execution of the batched lookup-permutation bodies (lookup.cuh) in capi_poly.cu's launch schedule
// (lookup_permuted_run), on the scratch of lk_plan: load every table, the bitonic network stage by stage (the global-stage body for every stride --
// the shared-memory kernel runs the same compare-exchanges), ranks + histogram, unconsumed flags, ONE exclusive scan over
// the whole call's concatenated segments, leftovers, then -- only when no lookup missed -- the fill and blinding rows.
// Never loaded by the halo2_b200 package; see tests/kernel_emul/README.md.
#include <cstring>
#include <vector>
#include "lookup.cuh"
using namespace h2;

// inputs / tables / out_in / out_tab: count x n canonical values; blinding: count x 2 rows canonical values or null.
// Returns H2_LK_NONE, or the lowest lookup with a miss (the outputs are then unchanged).
template <class P>
static uint32_t run_permuted(const uint8_t *inputs, const uint8_t *tables, uint32_t count, size_t n, size_t u, const uint8_t *blinding, size_t rows,
                             uint8_t *out_in, uint8_t *out_tab) {
    typedef LookupPermute<P> K;
    auto load = [&](const uint8_t *src, size_t len) {
        std::vector<fe> v(len);
        for (size_t i = 0; i < len; i++) { fe x; memcpy(x.v, src + 32 * i, 32); v[i] = fe_to_mont<P>(x); }
        return v;
    };
    std::vector<fe> in = load(inputs, count * n), tab = load(tables, count * n), oa = load(out_in, count * n), ot = load(out_tab, count * n);
    std::vector<fe> blind = blinding ? load(blinding, count * 2 * rows) : std::vector<fe>();
    uint32_t err = H2_LK_NONE;
    if (u) {
        const LkPlan plan = lk_plan(u, count);
        const uint64_t N = plan.N, w = plan.w;
        std::vector<fe> keys(plan.keys_end);
        std::vector<uint32_t> sc(plan.left - plan.sc, 0), left(plan.err - plan.left, 0);
        for (uint32_t b = 0; b < count; b++) {
            fe *kt = keys.data() + b * N;
            for (uint64_t i = 0; i < N; i++) K::load_body(tab.data() + b * n, u, kt, N, i);
            for (uint64_t size = 2; size <= N; size <<= 1)
                for (uint64_t stride = size / 2; stride >= 1; stride >>= 1)
                    for (uint64_t t = 0; t < N / 2; t++) K::global_stage_body(kt, N, size, stride, t);
        }
        for (uint32_t b = 0; b < count; b++)
            for (uint64_t i = 0; i < u; i++) {
                const uint32_t r = K::rank_body(in.data() + b * n, keys.data() + b * N, u, i);
                if (r == H2_LK_NONE) err = b < err ? b : err;
                else sc[b * w + r]++;
            }
        for (uint32_t b = 0; b < count; b++)
            for (uint64_t r = 0; r < w; r++) lk_unconsumed_body(sc.data() + b * w, u, sc.data() + (count + b) * w, r);
        uint32_t run = 0;                                          // exclusive scan, u32 arithmetic as on the device
        for (auto &x : sc) { const uint32_t v = x; x = run; run += v; }
        for (uint32_t b = 0; b < count; b++)
            for (uint64_t r = 0; r < u; r++) lk_leftover_body(sc.data() + (count + b) * w, u, left.data() + b * u, r);
        if (err != H2_LK_NONE) return err;
        for (uint32_t b = 0; b < count; b++) {
            for (uint64_t i = 0; i < u; i++)
                K::rank_fill_body(keys.data() + b * N, u, sc.data() + b * w, sc.data() + (count + b) * w, left.data() + b * u, oa.data() + b * n, ot.data() + b * n, i);
            if (blinding)
                for (uint64_t t = 0; t < rows; t++) K::blind_body(blind.data() + b * 2 * rows, rows, u, oa.data() + b * n, ot.data() + b * n, t);
        }
    }
    for (size_t i = 0; i < count * n; i++) {
        fe x = fe_from_mont<P>(oa[i]); memcpy(out_in + 32 * i, x.v, 32);
        x = fe_from_mont<P>(ot[i]); memcpy(out_tab + 32 * i, x.v, 32);
    }
    return err;
}
// lk_plan's fields in declaration order
extern "C" void emu_lookup_plan(uint64_t u, uint64_t count, uint64_t *out) {
    const LkPlan P = lk_plan(u, count);
    const uint64_t f[] = {P.N, P.w, P.keys, P.keys_end, P.sc, P.left, P.err, P.u32_end};
    memcpy(out, f, sizeof f);
}
// h2_poly_lookup_permuted: n = 2^k rows per lookup, u = n - rows usable ones, blinding = count x 2 rows values
extern "C" uint32_t emu_lookup_permuted(int field, const uint8_t *inputs, const uint8_t *tables, uint32_t count, size_t n, size_t u, const uint8_t *blinding,
                                        size_t rows, uint8_t *out_in, uint8_t *out_tab) {
    return field == 0 ? run_permuted<FpParams>(inputs, tables, count, n, u, blinding, rows, out_in, out_tab)
                      : run_permuted<FqParams>(inputs, tables, count, n, u, blinding, rows, out_in, out_tab);
}
