// TEST-ONLY serial execution of the lookup-permutation kernel bodies (lookup.cuh) on lk_plan's N and w: load, the bitonic
// network stage by stage (the global-stage body for every stride -- the shared-memory kernel runs the same
// compare-exchanges), run starts + lower bounds, the two scans, leftover scatter, fill.  Never loaded by the halo2_b200
// package; see tests/kernel_emul/README.md.
#include <cstring>
#include <vector>
#include "lookup.cuh"
using namespace h2;

template <class P> static int run_lookup(const uint8_t *input, const uint8_t *table, size_t n, size_t u, uint8_t *out_in, uint8_t *out_tab) {
    typedef LookupPermute<P> K;
    std::vector<fe> a(n), t(n), oa(n), ot(n);
    for (size_t i = 0; i < n; i++) {
        fe x; memcpy(x.v, input + 32 * i, 32); a[i] = fe_to_mont<P>(x);
        memcpy(x.v, table + 32 * i, 32); t[i] = fe_to_mont<P>(x);
        memcpy(x.v, out_in + 32 * i, 32); oa[i] = fe_to_mont<P>(x);      // the caller's markers: rows >= u must survive
        memcpy(x.v, out_tab + 32 * i, 32); ot[i] = fe_to_mont<P>(x);
    }
    if (u) {
        const LkPlan plan = lk_plan(u, 1);
        const uint64_t N = plan.N, w = plan.w;
        std::vector<fe> ka(N), kt(N), left(w);
        for (uint64_t i = 0; i < N; i++) { K::load_body(a.data(), u, ka.data(), N, i); K::load_body(t.data(), u, kt.data(), N, i); }
        for (auto *keys : {ka.data(), kt.data()})
            for (uint64_t size = 2; size <= N; size <<= 1)
                for (uint64_t stride = size / 2; stride >= 1; stride >>= 1)
                    for (uint64_t th = 0; th < N / 2; th++) K::global_stage_body(keys, N, size, stride, th);
        std::vector<uint32_t> first(w, 0), unc(w, 0), fs(w), us(w);
        for (size_t i = 0; i < u; i++) unc[i] = 1;
        uint32_t err = 0;
        for (uint64_t r = 0; r < u; r++) K::first_body(ka.data(), kt.data(), u, first.data(), unc.data(), &err, oa.data(), ot.data(), r);
        if (err) return 1;
        uint32_t run = 0;
        for (size_t i = 0; i <= u; i++) { fs[i] = run; run += first[i]; }
        run = 0;
        for (size_t i = 0; i <= u; i++) { us[i] = run; run += unc[i]; }
        for (uint64_t i = 0; i < u; i++) K::leftover_body(kt.data(), u, unc.data(), us.data(), left.data(), i);
        for (uint64_t r = 0; r < u; r++) K::fill_body(u, first.data(), fs.data(), left.data(), ot.data(), r);
    }
    for (size_t i = 0; i < n; i++) {
        fe x = fe_from_mont<P>(oa[i]); memcpy(out_in + 32 * i, x.v, 32);
        x = fe_from_mont<P>(ot[i]); memcpy(out_tab + 32 * i, x.v, 32);
    }
    return 0;
}
// canonical 32-byte values; out_in / out_tab hold n values on entry (markers) and the permuted columns in their first u rows on
// exit; returns 1 where the reference fails (an input value missing from the table)
extern "C" int emu_lookup_permute(int field, const uint8_t *input, const uint8_t *table, size_t n, size_t u, uint8_t *out_in, uint8_t *out_tab) {
    return field == 0 ? run_lookup<FpParams>(input, table, n, u, out_in, out_tab) : run_lookup<FqParams>(input, table, n, u, out_in, out_tab);
}
