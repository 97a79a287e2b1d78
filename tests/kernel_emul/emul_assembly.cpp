// TEST-ONLY serial execution of the copy-cycle kernels (assembly.cuh) in the order and with the launch shapes of
// capi_poly.cu's assembly_run, with its round limit (as_round_limit) but separate vectors where the device carves
// as_edge_layout and as_slot_layout; the scans are plain exclusive scans, as the scan kernels of msm.cuh compute them.
#include <algorithm>
#include <vector>
#include "assembly.cuh"
using namespace h2;

static void scan(uint32_t *a, uint64_t n) {                      // exclusive, in place
    uint32_t run = 0;
    for (uint64_t i = 0; i < n; i++) { const uint32_t v = a[i]; a[i] = run; run += v; }
}
template <class F> static void grid(uint64_t threads, uint32_t block, F body) {   // every thread of the launched grid
    const uint64_t all = (threads + block - 1) / block * block;
    for (uint64_t t = 0; t < all; t++) body(t);
}

// map_out: cols * 2^k (column, row) pairs.  Returns 0, 1 for a bad copy (*bad = 2 i for a column, 2 i + 1 for a row of the
// first bad copy i) or 2 when the spanning forest would take more than floor(log2 cells) Borůvka rounds; *rounds_out =
// the rounds run, *forest_out = |F|.
extern "C" int emu_assembly(const uint32_t *copies, uint64_t m, uint32_t cols, uint32_t k, uint32_t *map_out, unsigned long long *bad,
                            uint32_t *rounds_out, uint32_t *forest_out) {
    const uint64_t N = (uint64_t)cols << k;
    std::vector<uint32_t> ea(m), eb(m), flag(m + 1), live0(m), live1(m), ra(m), rb(m), keep(m + 1, 0), fl(m);
    uint2 *map = reinterpret_cast<uint2 *>(map_out);
    *bad = ~0ull;
    *rounds_out = *forest_out = 0;
    if (m) grid(m + 1, 256, [&](uint64_t i) { AssemblyOps::encode_body(copies, (uint32_t)m, cols, k, ea.data(), eb.data(), flag.data(), bad, i); });
    if (*bad != ~0ull) return 1;
    grid(N, 256, [&](uint64_t v) { AssemblyOps::identity_body(map, N, k, v); });
    if (m == 0) return 0;
    scan(flag.data(), m + 1);
    uint32_t L = flag[m];
    grid(m, 256, [&](uint64_t e) { AssemblyOps::compact_body(flag.data(), (uint32_t)m, nullptr, live0.data(), e); });
    if (L) {
        std::vector<uint32_t> comp(N), best(N);
        grid(N, 256, [&](uint64_t v) { AssemblyOps::iota_body(comp.data(), N, v); });
        const uint32_t limit = as_round_limit(N);
        uint32_t *live[2] = {live0.data(), live1.data()};
        for (uint32_t round = 0, cur = 0; L; round++, cur ^= 1) {
            if (round == limit) return 2;
            const uint32_t *lv = live[cur];
            grid(L, 256, [&](uint64_t e) { AssemblyOps::roots_body(lv, L, ea.data(), eb.data(), comp.data(), ra.data(), rb.data(), best.data(), e); });
            grid(L, 256, [&](uint64_t e) { AssemblyOps::best_body(lv, L, ra.data(), rb.data(), best.data(), e); });
            grid(L, 256, [&](uint64_t e) { AssemblyOps::hook_body(lv, L, ra.data(), rb.data(), best.data(), comp.data(), keep.data(), e); });
            for (uint32_t changed = 1; changed;) {
                changed = 0;
                grid(N, 256, [&](uint64_t v) { AssemblyOps::jump_body(comp.data(), N, &changed, v); });
            }
            grid(L + 1, 256, [&](uint64_t e) { AssemblyOps::split_body(lv, L, ea.data(), eb.data(), comp.data(), flag.data(), e); });
            scan(flag.data(), L + 1);
            grid(L, 256, [&](uint64_t e) { AssemblyOps::compact_body(flag.data(), L, lv, live[cur ^ 1], e); });
            L = flag[L];
            *rounds_out = round + 1;
        }
    }
    scan(keep.data(), m + 1);
    const uint32_t q = keep[m];
    *forest_out = q;
    if (q == 0) return 0;
    grid(m, 256, [&](uint64_t i) { AssemblyOps::compact_body(keep.data(), (uint32_t)m, nullptr, fl.data(), i); });
    const uint64_t S = 2ull * q, ntiles = as_slot_layout(S).ntiles;
    std::vector<uint32_t> scell(S), order0(S), order1(S), nxt0(S), nxt1(S), counts(H2_AS_TILE * ntiles + 1);
    uint32_t *order[2] = {order0.data(), order1.data()}, *nxt[2] = {nxt0.data(), nxt1.data()};
    grid(S, 256, [&](uint64_t s) { AssemblyOps::slots_body(fl.data(), S, ea.data(), eb.data(), scell.data(), order[0], s); });
    uint32_t o = 0;
    for (uint32_t shift = 0; shift == 0 || ((N - 1) >> shift); shift += H2_AS_DIGIT_BITS, o ^= 1) {
        for (uint64_t tile = 0; tile < ntiles; tile++) {                  // as_radix_hist_kernel, one block per tile
            uint32_t cnt[H2_AS_TILE] = {};
            for (uint32_t t = 0; t < H2_AS_TILE; t++) AssemblyOps::radix_hist_body(order[o], S, scell.data(), shift, cnt, tile, t);
            for (uint32_t d = 0; d < H2_AS_TILE; d++) counts[d * ntiles + tile] = cnt[d];
        }
        counts[H2_AS_TILE * ntiles] = 0;
        scan(counts.data(), H2_AS_TILE * ntiles + 1);
        for (uint64_t tile = 0; tile < ntiles; tile++) {                  // as_radix_scatter_kernel
            uint32_t dig[H2_AS_TILE];
            for (uint32_t t = 0; t < H2_AS_TILE; t++) {
                const uint64_t idx = tile * H2_AS_TILE + t;
                dig[t] = idx < S ? AssemblyOps::digit(scell[order[o][idx]], shift) : H2_AS_NONE;
            }
            for (uint32_t t = 0; t < H2_AS_TILE; t++) AssemblyOps::radix_scatter_body(order[o], S, counts.data(), ntiles, dig, tile, t, order[o ^ 1]);
        }
    }
    grid(S, 256, [&](uint64_t p) { AssemblyOps::succ_body(order[o], S, scell.data(), nxt[0], p); });
    uint32_t t = 0;
    for (uint64_t len = 1; len <= S; len <<= 1, t ^= 1)
        grid(S, 256, [&](uint64_t s) { AssemblyOps::jump_slots_body(nxt[t], nxt[t ^ 1], S, s); });
    grid(S, 256, [&](uint64_t p) { AssemblyOps::final_body(order[o], S, scell.data(), nxt[t], k, map, p); });
    return 0;
}

// The scratch layouts' fields in declaration order: as_edge_layout(m) into edge (13 values), as_slot_layout(S) into slot (8)
extern "C" void emu_assembly_layouts(uint64_t m, uint64_t S, uint64_t *edge, uint64_t *slot) {
    const AsEdgeLayout E = as_edge_layout(m);
    const uint64_t e[] = {E.err, E.changed, E.copies, E.ea, E.eb, E.flag, E.live[0], E.live[1], E.ra, E.rb, E.keep, E.fl, E.end};
    const AsSlotLayout Q = as_slot_layout(S);
    const uint64_t q[] = {Q.ntiles, Q.scell, Q.order[0], Q.order[1], Q.nxt[0], Q.nxt[1], Q.counts, Q.end};
    std::copy(e, e + 13, edge);
    std::copy(q, q + 8, slot);
}
