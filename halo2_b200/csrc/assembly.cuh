// K20: the permutation argument's copy cycles from the list of copy constraints, on the device.
//
//   Assembly::copy         /root/reference/halo2_proofs/src/plonk/permutation/keygen.rs:45-100
//
// The reference replays the copies one by one, merging cycles.  Its final `mapping` has a closed form (DESIGN.md K20):
//   1. only the final swap of `copy` changes `mapping`: swapping entries l and r is M <- M o (l r);
//   2. a copy is applied iff its two cells are not yet connected by the copies before it, so the applied copies are the
//      minimum spanning forest F of the copy graph with weight = copy index (Kruskal's forest);
//   3. M is the product of F's transpositions in copy order: M(v) is the end of a walk that leaves v by its largest F-edge
//      and, at every cell reached, leaves by the largest F-edge below the one it arrived by;
//   4. that walk is a successor function on slots (cell, F-edge at the cell), so pointer jumping ends every walk at once.
// Here: encode and check the copies; F by Borůvka rounds (weights distinct, so F is unique whatever the thread schedule);
// the 2|F| slots stably radix-sorted by cell, so every cell's slots stay in copy order whatever its degree; successor and
// pointer jumping over the slots; the mapping as (column, row) pairs for the sigma kernel of keygen.cuh.
//
// A cell (c, r) is the id c * 2^k + r < cols * 2^k < 2^32; a copy is its index in synthesis order.  The per-thread bodies
// compile for the host emulation (tests/kernel_emul/emul_assembly.cpp), where the atomics are plain read-modify-writes.
#pragma once
#include "field.cuh"

namespace h2 {

#define H2_AS_NONE 0xFFFFFFFFu
#define H2_AS_TILE 256                   // items per radix-sort tile = the 256 digit values of one pass
#define H2_AS_DIGIT_BITS 8

H2_HD void as_atomic_min(uint32_t *p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}
H2_HD void as_atomic_min64(unsigned long long *p, unsigned long long v) {
#if defined(__CUDA_ARCH__)
    atomicMin(p, v);
#else
    if (v < *p) *p = v;
#endif
}
H2_HD void as_atomic_inc(uint32_t *p) {
#if defined(__CUDA_ARCH__)
    atomicAdd(p, 1u);
#else
    *p += 1;
#endif
}

struct AssemblyOps {
    // ---- 1. encode and check: copy i = copies[4 i .. 4 i + 3] = (lc, lr, rc, rr) -> cells ea[i], eb[i];
    // flag[i] = 1 for a copy of two different cells (flag[m] = 0, for the scan); a bad copy puts 2 i (a column outside the
    // permutation, Error::ColumnNotInPermutation, checked first as the reference does) or 2 i + 1 (a row outside the
    // domain, Error::BoundsFailure) into the error word by min, so the first bad copy is the one reported
    static H2_HD void encode_body(const uint32_t *copies, uint32_t m, uint32_t cols, uint32_t k, uint32_t *ea, uint32_t *eb, uint32_t *flag,
                                  unsigned long long *err, uint64_t i) {
        if (i > m) return;
        if (i == m) { flag[m] = 0; return; }
        const uint32_t lc = copies[4 * i], lr = copies[4 * i + 1], rc = copies[4 * i + 2], rr = copies[4 * i + 3];
        if (lc >= cols || rc >= cols) { as_atomic_min64(err, 2ull * i); flag[i] = 0; return; }
        if ((uint64_t)lr >> k || (uint64_t)rr >> k) { as_atomic_min64(err, 2ull * i + 1); flag[i] = 0; return; }
        const uint32_t a = (lc << k) | lr, b = (rc << k) | rr;
        ea[i] = a;
        eb[i] = b;
        flag[i] = a != b;
    }
    // stream compaction after an exclusive scan of n + 1 flags: item e was flagged iff scan[e + 1] != scan[e]
    static H2_HD void compact_body(const uint32_t *scan, uint32_t n, const uint32_t *in, uint32_t *out, uint64_t e) {
        if (e < n && scan[e + 1] != scan[e]) out[scan[e]] = in ? in[e] : (uint32_t)e;
    }
    static H2_HD void iota_body(uint32_t *a, uint64_t n, uint64_t v) {
        if (v < n) a[v] = (uint32_t)v;
    }

    // ---- 2. Borůvka rounds over the live copies live[0 .. L) (each joins two different components; comp[] is a star forest)
    // the two endpoint components of every live copy, and their `best` reset
    static H2_HD void roots_body(const uint32_t *live, uint32_t L, const uint32_t *ea, const uint32_t *eb, const uint32_t *comp, uint32_t *ra,
                                 uint32_t *rb, uint32_t *best, uint64_t e) {
        if (e >= L) return;
        const uint32_t i = live[e], a = comp[ea[i]], b = comp[eb[i]];
        ra[e] = a;
        rb[e] = b;
        best[a] = H2_AS_NONE;
        best[b] = H2_AS_NONE;
    }
    // every component's lightest live copy (the smallest index)
    static H2_HD void best_body(const uint32_t *live, uint32_t L, const uint32_t *ra, const uint32_t *rb, uint32_t *best, uint64_t e) {
        if (e >= L) return;
        const uint32_t i = live[e];
        as_atomic_min(best + ra[e], i);
        as_atomic_min(best + rb[e], i);
    }
    // a component hooks to the other end of its lightest copy, which joins F; two components that chose the same copy
    // (a mutual pair) hook the larger id to the smaller.  Reads ra / rb / best only, so no thread sees another's hook.
    static H2_HD void hook_body(const uint32_t *live, uint32_t L, const uint32_t *ra, const uint32_t *rb, const uint32_t *best, uint32_t *comp,
                                uint32_t *keep, uint64_t e) {
        if (e >= L) return;
        const uint32_t i = live[e], a = ra[e], b = rb[e];
        const bool ca = best[a] == i, cb = best[b] == i;
        if (!ca && !cb) return;
        keep[i] = 1;
        if (ca && cb) {
            if (a < b) comp[b] = a;
            else comp[a] = b;
        } else if (ca) comp[a] = b;
        else comp[b] = a;
    }
    // pointer jumping on comp[] in place: every pointer only ever moves to an ancestor, so the races are benign
    static H2_HD void jump_body(uint32_t *comp, uint64_t n, uint32_t *changed, uint64_t v) {
        if (v >= n) return;
        const uint32_t c = comp[v], cc = comp[c];
        if (cc != c) { comp[v] = cc; *changed = 1; }
    }
    // flag[e] = 1 for a live copy whose ends are still in different components (flag[L] = 0, for the scan)
    static H2_HD void split_body(const uint32_t *live, uint32_t L, const uint32_t *ea, const uint32_t *eb, const uint32_t *comp, uint32_t *flag,
                                 uint64_t e) {
        if (e > L) return;
        if (e == L) { flag[L] = 0; return; }
        const uint32_t i = live[e];
        flag[e] = comp[ea[i]] != comp[eb[i]];
    }

    // ---- 3. slots: slot 2 j / 2 j + 1 is the left / right end of F's j-th copy fl[j]; slot order is copy order
    static H2_HD void slots_body(const uint32_t *fl, uint64_t S, const uint32_t *ea, const uint32_t *eb, uint32_t *scell, uint32_t *order, uint64_t s) {
        if (s >= S) return;
        const uint32_t i = fl[s >> 1];
        scell[s] = (s & 1) ? eb[i] : ea[i];
        order[s] = (uint32_t)s;
    }
    static H2_HD uint32_t digit(uint32_t cell, uint32_t shift) { return (cell >> shift) & ((1u << H2_AS_DIGIT_BITS) - 1); }
    // one LSD pass of a stable radix sort of order[] by scell[]: count the digits of one tile ...
    static H2_HD void radix_hist_body(const uint32_t *order, uint64_t S, const uint32_t *scell, uint32_t shift, uint32_t *tile_cnt, uint64_t tile,
                                      uint32_t t) {
        const uint64_t idx = tile * H2_AS_TILE + t;
        if (idx < S) as_atomic_inc(tile_cnt + digit(scell[order[idx]], shift));
    }
    // ... and, after the exclusive scan of counts[digit * ntiles + tile], place every item at its digit's offset plus its
    // rank among the tile's earlier items of the same digit (dig[] = the tile's digits), which keeps the sort stable
    static H2_HD void radix_scatter_body(const uint32_t *order, uint64_t S, const uint32_t *counts, uint64_t ntiles, const uint32_t *dig, uint64_t tile,
                                         uint32_t t, uint32_t *out) {
        const uint64_t idx = tile * H2_AS_TILE + t;
        if (idx >= S) return;
        const uint32_t d = dig[t];
        uint32_t rank = 0;
        for (uint32_t u = 0; u < t; u++) rank += dig[u] == d;
        out[counts[d * ntiles + tile] + rank] = order[idx];
    }
    // ---- 4. the walk's successor: arriving at cell x by slot s, leave by the previous slot of x's list (the largest index
    // below s's), i.e. continue at its twin; the first slot of a list ends the walk (nxt[s] = s)
    static H2_HD void succ_body(const uint32_t *order, uint64_t S, const uint32_t *scell, uint32_t *nxt, uint64_t p) {
        if (p >= S) return;
        const uint32_t s = order[p];
        nxt[s] = (p > 0 && scell[order[p - 1]] == scell[s]) ? (order[p - 1] ^ 1u) : s;
    }
    static H2_HD void jump_slots_body(const uint32_t *in, uint32_t *out, uint64_t S, uint64_t s) {
        if (s < S) out[s] = in[in[s]];
    }
    // ---- 5. the mapping: every cell to itself ...
    static H2_HD void identity_body(uint2 *map, uint64_t n, uint32_t k, uint64_t v) {
        if (v < n) map[v] = make_uint2((uint32_t)(v >> k), (uint32_t)(v & ((1ull << k) - 1)));
    }
    // ... and a cell with F-edges (at the last slot of its list) to the end of the walk that starts at that slot's twin
    static H2_HD void final_body(const uint32_t *order, uint64_t S, const uint32_t *scell, const uint32_t *term, uint32_t k, uint2 *map, uint64_t p) {
        if (p >= S) return;
        const uint32_t s = order[p], x = scell[s];
        if (p + 1 < S && scell[order[p + 1]] == x) return;
        const uint32_t y = scell[term[s ^ 1u]];
        map[x] = make_uint2(y >> k, y & (uint32_t)((1ull << k) - 1));
    }
};

// After r Borůvka rounds a component with a live copy has >= 2^r cells, so F takes at most floor(log2 cells) rounds.
inline uint32_t as_round_limit(uint64_t cells) {
    uint32_t r = 0;
    while ((2ull << r) <= cells) r++;
    return r;
}
// The per-copy scratch (as_edge) of m copies, in u32 words: the error word (u64), `changed` (the pointer-jumping flag, in
// a u64 slot), the copies (4 words each), ea, eb, flag (m + 1 words: the scan's total), the two live lists, ra, rb, keep
// (m + 1) and F.
struct AsEdgeLayout {
    uint64_t err, changed, copies, ea, eb, flag, live[2], ra, rb, keep, fl, end;
};
inline AsEdgeLayout as_edge_layout(uint64_t m) {
    AsEdgeLayout A{};
    auto take = [&](uint64_t words) { const uint64_t at = A.end; A.end += words; return at; };
    A.err = take(2);
    A.changed = take(2);
    A.copies = take(4 * m);
    A.ea = take(m);
    A.eb = take(m);
    A.flag = take(m + 1);
    A.live[0] = take(m);
    A.live[1] = take(m);
    A.ra = take(m);
    A.rb = take(m);
    A.keep = take(m + 1);
    A.fl = take(m);
    return A;
}
// The per-slot scratch (as_slot) of S slots, in u32 words: the slots' cells, order and nxt (two buffers each) and the
// radix sort's digit counts, H2_AS_TILE per tile and the scan's total.
struct AsSlotLayout {
    uint64_t ntiles, scell, order[2], nxt[2], counts, end;
};
inline AsSlotLayout as_slot_layout(uint64_t S) {
    AsSlotLayout A{};
    auto take = [&](uint64_t words) { const uint64_t at = A.end; A.end += words; return at; };
    A.ntiles = (S + H2_AS_TILE - 1) / H2_AS_TILE;
    A.scell = take(S);
    A.order[0] = take(S);
    A.order[1] = take(S);
    A.nxt[0] = take(S);
    A.nxt[1] = take(S);
    A.counts = take(H2_AS_TILE * A.ntiles + 1);
    return A;
}

#if defined(__CUDACC__)
#define H2_AS_TID ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x)
__global__ void __launch_bounds__(256) as_encode_kernel(const uint32_t *copies, uint32_t m, uint32_t cols, uint32_t k, uint32_t *ea, uint32_t *eb,
                                                        uint32_t *flag, unsigned long long *err) {
    AssemblyOps::encode_body(copies, m, cols, k, ea, eb, flag, err, H2_AS_TID);
}
__global__ void __launch_bounds__(256) as_compact_kernel(const uint32_t *scan, uint32_t n, const uint32_t *in, uint32_t *out) {
    AssemblyOps::compact_body(scan, n, in, out, H2_AS_TID);
}
__global__ void __launch_bounds__(256) as_iota_kernel(uint32_t *a, uint64_t n) { AssemblyOps::iota_body(a, n, H2_AS_TID); }
__global__ void __launch_bounds__(256) as_roots_kernel(const uint32_t *live, uint32_t L, const uint32_t *ea, const uint32_t *eb, const uint32_t *comp,
                                                       uint32_t *ra, uint32_t *rb, uint32_t *best) {
    AssemblyOps::roots_body(live, L, ea, eb, comp, ra, rb, best, H2_AS_TID);
}
__global__ void __launch_bounds__(256) as_best_kernel(const uint32_t *live, uint32_t L, const uint32_t *ra, const uint32_t *rb, uint32_t *best) {
    AssemblyOps::best_body(live, L, ra, rb, best, H2_AS_TID);
}
__global__ void __launch_bounds__(256) as_hook_kernel(const uint32_t *live, uint32_t L, const uint32_t *ra, const uint32_t *rb, const uint32_t *best,
                                                      uint32_t *comp, uint32_t *keep) {
    AssemblyOps::hook_body(live, L, ra, rb, best, comp, keep, H2_AS_TID);
}
__global__ void __launch_bounds__(256) as_jump_kernel(uint32_t *comp, uint64_t n, uint32_t *changed) {
    AssemblyOps::jump_body(comp, n, changed, H2_AS_TID);
}
__global__ void __launch_bounds__(256) as_split_kernel(const uint32_t *live, uint32_t L, const uint32_t *ea, const uint32_t *eb, const uint32_t *comp,
                                                       uint32_t *flag) {
    AssemblyOps::split_body(live, L, ea, eb, comp, flag, H2_AS_TID);
}
__global__ void __launch_bounds__(256) as_slots_kernel(const uint32_t *fl, uint64_t S, const uint32_t *ea, const uint32_t *eb, uint32_t *scell,
                                                       uint32_t *order) {
    AssemblyOps::slots_body(fl, S, ea, eb, scell, order, H2_AS_TID);
}
// counts[digit * ntiles + tile] for one pass; counts[256 ntiles] = 0 so the scan leaves the total there
__global__ void __launch_bounds__(H2_AS_TILE) as_radix_hist_kernel(const uint32_t *order, uint64_t S, const uint32_t *scell, uint32_t shift,
                                                                   uint64_t ntiles, uint32_t *counts) {
    __shared__ uint32_t cnt[H2_AS_TILE];
    cnt[threadIdx.x] = 0;
    __syncthreads();
    AssemblyOps::radix_hist_body(order, S, scell, shift, cnt, blockIdx.x, threadIdx.x);
    __syncthreads();
    counts[threadIdx.x * ntiles + blockIdx.x] = cnt[threadIdx.x];
    if (blockIdx.x == 0 && threadIdx.x == 0) counts[H2_AS_TILE * ntiles] = 0;
}
__global__ void __launch_bounds__(H2_AS_TILE) as_radix_scatter_kernel(const uint32_t *order, uint64_t S, const uint32_t *scell, uint32_t shift,
                                                                      const uint32_t *counts, uint64_t ntiles, uint32_t *out) {
    __shared__ uint32_t dig[H2_AS_TILE];
    const uint64_t idx = (uint64_t)blockIdx.x * H2_AS_TILE + threadIdx.x;
    dig[threadIdx.x] = idx < S ? AssemblyOps::digit(scell[order[idx]], shift) : H2_AS_NONE;
    __syncthreads();
    AssemblyOps::radix_scatter_body(order, S, counts, ntiles, dig, blockIdx.x, threadIdx.x, out);
}
__global__ void __launch_bounds__(256) as_succ_kernel(const uint32_t *order, uint64_t S, const uint32_t *scell, uint32_t *nxt) {
    AssemblyOps::succ_body(order, S, scell, nxt, H2_AS_TID);
}
__global__ void __launch_bounds__(256) as_jump_slots_kernel(const uint32_t *in, uint32_t *out, uint64_t S) {
    AssemblyOps::jump_slots_body(in, out, S, H2_AS_TID);
}
__global__ void __launch_bounds__(256) as_identity_kernel(uint2 *map, uint64_t n, uint32_t k) { AssemblyOps::identity_body(map, n, k, H2_AS_TID); }
__global__ void __launch_bounds__(256) as_final_kernel(const uint32_t *order, uint64_t S, const uint32_t *scell, const uint32_t *term, uint32_t k,
                                                       uint2 *map) {
    AssemblyOps::final_body(order, S, scell, term, k, map, H2_AS_TID);
}
#undef H2_AS_TID
#endif

}  // namespace h2
