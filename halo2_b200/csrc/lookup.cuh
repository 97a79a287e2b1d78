// The lookup argument's permuted columns on resident polynomials, every lookup of a call at once (grid.y = lookup).
//
// Replaces permute_expression_pair (/root/reference/halo2_proofs/src/plonk/lookup/prover.rs:563-647), the one step of the
// prover's middle section that is neither an FFT, an MSM nor an elementwise program: given the compressed input column A and
// table column S over the usable rows [0, u) it returns
//   A' = A sorted (ff's Ord: the canonical integers, :577-581), and
//   S' with S'[r] = A'[r] on the first row of every run of equal values in A' (:595-603; the value must occur in S, else
//      Error::ConstraintSystemFailure, :605-608), the other rows filled with the table values that are left over, smallest
//      first, handed to the repeated rows from the LAST one down (`repeated_input_rows.pop()`, :617-622).
// The reference does this with a sort and a BTreeMap on one core.  Here only the table is sorted (bitonic, 256-bit canonical
// keys: shared memory below 1024 keys, one launch per global stage above).  The input is ordered by rank instead of by a
// second sort: r = the lower bound of an input value in the sorted table T is strictly increasing on the values T holds, so
//   cnt[r] = #inputs of rank r (warp-aggregated histogram: most rows of a real input hold one value), off = its exclusive scan;
//   A'[i] = T[r] for the last r with off[r] <= i;  the run of rank r starts at row off[r], where S' = T[r];
//   T[r] is left over exactly when cnt[r] == 0 (duplicates too: the search always lands on the first of them), and the j-th
//   repeated row takes leftover[L - 1 - j].
// Optionally the blinding rows [u, n) (:622-627) take the caller's random values.  Nothing is written to an output unless
// every lookup of the call found all its input values: the miss is found (and its lowest lookup index recorded) by the
// histogram kernel, and the one kernel that writes the outputs runs after it and checks the error word first.
#pragma once
#include "field.cuh"

namespace h2 {

// lexicographic order of canonical (non-Montgomery) elements = order of the integers
H2_HD bool fe_canon_lt(const fe &a, const fe &b) {
    for (int i = 7; i >= 0; i--) {
        if (a.v[i] != b.v[i]) return a.v[i] < b.v[i];
    }
    return false;
}

#define H2_LK_BLOCK_LOG 10u           // keys per shared-memory block of the bitonic sort
#define H2_LK_NONE 0xffffffffu        // the error word when no lookup missed; the rank of an input value the table lacks

// One call: `count` lookups of u usable rows, keys padded to N = 2^m >= u per lookup.  Lookup b's arrays:
//   keys  fe  [b N, (b + 1) N)             its table, canonical, sorted
//   sc    u32 [b w, (b + 1) w), w = u + 1  cnt, then (after the scan) off, of the whole call's concatenated scan
//   sc    u32 [(count + b) w, ...)         unconsumed flags, then their scan
//   left  u32 [b u, (b + 1) u)             table ranks of the leftover values, ascending
// The scan runs once over all 2 count w words; a lookup's values are differences from its segment's first word (exact in
// u32 arithmetic, every segment sums to at most u < 2^31).
// The plan of one call: N and w, the element offsets of keys (in lk_keys), of sc, left and the error word (in lk_u32), and
// where each pool's part ends.
struct LkPlan {
    uint64_t N, w;
    uint64_t keys, keys_end;                   // fe
    uint64_t sc, left, err, u32_end;           // u32
};
inline LkPlan lk_plan(uint64_t u, uint64_t count) {
    LkPlan P{};
    P.N = 2;
    while (P.N < u) P.N <<= 1;
    P.w = u + 1;
    P.keys = 0;
    P.keys_end = count * P.N;
    auto take = [&](uint64_t words) { const uint64_t at = P.u32_end; P.u32_end += words; return at; };
    P.sc = take(2 * P.w * count);
    P.left = take(u * count);
    P.err = take(1);
    return P;
}
// unc[r] = 1 when table rank r < u is consumed by no input row (cnt[r] == 0); unc[u] = 0 closes the segment
H2_HD void lk_unconsumed_body(const uint32_t *cnt, uint64_t u, uint32_t *unc, uint64_t r) {
    if (r <= u) unc[r] = (r < u && cnt[r] == 0) ? 1u : 0u;
}
// after the scan (uscan = the lookup's segment of scanned flags): left[q] = the rank of the q-th unconsumed table value
H2_HD void lk_leftover_body(const uint32_t *uscan, uint64_t u, uint32_t *left, uint64_t r) {
    if (r >= u) return;
    const uint32_t q = uscan[r] - uscan[0];
    if (uscan[r + 1] - uscan[0] != q) left[q] = (uint32_t)r;
}
template <class P> struct LookupPermute {
    // keys[i] = canonical src[i] for i < u, the all-ones sentinel (> every field element) up to the power of two N
    static H2_HD void load_body(const fe *src, uint64_t u, fe *keys, uint64_t N, uint64_t i) {
        if (i >= N) return;
        fe x;
        if (i < u) x = fe_from_mont<P>(fe_load(src + i));
        else for (int k = 0; k < 8; k++) x.v[k] = 0xffffffffu;
        fe_store(keys + i, x);
    }
    // one compare-exchange of the bitonic network: pair (i, i + stride) of the merge of `size` keys that i lies in
    static H2_HD void global_stage_body(fe *keys, uint64_t N, uint64_t size, uint64_t stride, uint64_t t) {
        if (t >= N / 2) return;
        const uint64_t i = (t / stride) * 2 * stride + (t % stride), j = i + stride;
        fe a = fe_load(keys + i), b = fe_load(keys + j);
        const bool before = fe_canon_lt(b, a);
        if (before == ((i & size) == 0)) { fe_store(keys + i, b); fe_store(keys + j, a); }
    }
    // the rank of input row i: the lower bound of its value in the sorted table kt[0, u), H2_LK_NONE when the table lacks it
    static H2_HD uint32_t rank_body(const fe *src, const fe *kt, uint64_t u, uint64_t i) {
        const fe v = fe_from_mont<P>(fe_load(src + i));
        uint64_t lo = 0, hi = u;
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if (fe_canon_lt(fe_load(kt + mid), v)) lo = mid + 1; else hi = mid;
        }
        return (lo < u && fe_eq(fe_load(kt + lo), v)) ? (uint32_t)lo : H2_LK_NONE;
    }
    // row i < u of both outputs (Montgomery); off / uscan are the lookup's scanned segments, kt its sorted table
    static H2_HD void rank_fill_body(const fe *kt, uint64_t u, const uint32_t *off, const uint32_t *uscan, const uint32_t *left, fe *out_input,
                                     fe *out_table, uint64_t i) {
        const uint32_t o0 = off[0], u0 = uscan[0];
        uint64_t lo = 0, hi = u;                                   // the last r with off[r] <= i: upper bound of i in off[0, u], less one
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if ((uint64_t)(off[mid] - o0) <= i) lo = mid + 1; else hi = mid;
        }
        const uint64_t r = lo - 1;
        const fe tr = fe_to_mont<P>(fe_load(kt + r));
        fe_store(out_input + i, tr);
        if ((uint64_t)(off[r] - o0) == i) { fe_store(out_table + i, tr); return; }
        // rows before i that start a run: one per consumed rank <= r (rank r's own run starts before i)
        const uint64_t firsts_before = r + 1 - (uint64_t)(uscan[r] - u0), j = i - firsts_before, L = uscan[u] - u0;
        fe_store(out_table + i, fe_to_mont<P>(fe_load(kt + left[L - 1 - j])));
    }
    // blinding row u + t of both outputs: blind = (bf + 1) input values then (bf + 1) table values, Montgomery
    static H2_HD void blind_body(const fe *blind, uint64_t rows, uint64_t u, fe *out_input, fe *out_table, uint64_t t) {
        if (t >= rows) return;
        fe_store(out_input + u + t, fe_load(blind + t));
        fe_store(out_table + u + t, fe_load(blind + rows + t));
    }
    // K17's two-sort form: the input sorted like the table, run starts found by comparing neighbours.  No kernel runs it; the
    // host emulation does (tests/kernel_emul/emul_lookup.cpp), as a second restatement whose bytes the rank form above must
    // equal (tests/test_lookup_permuted_oracle.py).
    // rows r < u of the sorted input: out_input[r] = A'[r]; on the first row of a run also out_table[r] = A'[r] and the
    // table value it consumes is marked (lower bound in the sorted table; a miss raises *err).  first[r] = 1 / 0.
    static H2_HD void first_body(const fe *ka, const fe *kt, uint64_t u, uint32_t *first, uint32_t *unconsumed, uint32_t *err, fe *out_input,
                                 fe *out_table, uint64_t r) {
        if (r >= u) return;
        const fe v = fe_load(ka + r);
        fe_store(out_input + r, fe_to_mont<P>(v));
        bool is_first = r == 0;
        if (!is_first) is_first = !fe_eq(v, fe_load(ka + r - 1));
        first[r] = is_first ? 1u : 0u;
        if (!is_first) return;
        fe_store(out_table + r, fe_to_mont<P>(v));
        uint64_t lo = 0, hi = u;                                   // lower bound of v in kt[0, u)
        while (lo < hi) {
            const uint64_t mid = (lo + hi) >> 1;
            if (fe_canon_lt(fe_load(kt + mid), v)) lo = mid + 1; else hi = mid;
        }
        if (lo >= u || !fe_eq(fe_load(kt + lo), v)) { *err = 1u; return; }
        unconsumed[lo] = 0u;                                       // distinct values have distinct lower bounds: no race
    }
    // leftover[rank] = the rank-th unconsumed table value (ranks from the exclusive scan of `unconsumed`)
    static H2_HD void leftover_body(const fe *kt, uint64_t u, const uint32_t *unconsumed_flag, const uint32_t *rank, fe *leftover, uint64_t i) {
        if (i < u && unconsumed_flag[i]) fe_store(leftover + rank[i], fe_load(kt + i));
    }
    // repeated rows take the leftovers from the back: the j-th repeated row (j = r - firsts_before[r]) gets leftover[L - 1 - j]
    static H2_HD void fill_body(uint64_t u, const uint32_t *first_flag, const uint32_t *firsts_before, const fe *leftover, fe *out_table, uint64_t r) {
        if (r >= u || first_flag[r]) return;
        const uint64_t total_first = firsts_before[u], L = u - total_first, j = r - firsts_before[r];
        fe_store(out_table + r, fe_to_mont<P>(fe_load(leftover + (L - 1 - j))));
    }
};

#if defined(__CUDACC__)
// Lookup blockIdx.y's columns: the pointer arrays hold count entries each
struct LkCols {
    const fe *const *in;
    const fe *const *tab;
    fe *const *out_in;
    fe *const *out_tab;
    const fe *blind;                  // count x 2 (bf + 1) Montgomery values, or nullptr
};
template <class P> __global__ void __launch_bounds__(256) lk_load_kernel(LkCols c, uint64_t u, fe *keys, uint64_t N) {
    LookupPermute<P>::load_body(c.tab[blockIdx.y], u, keys + blockIdx.y * N, N, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
// Shared-memory part of the bitonic sort on a block of 2^H2_LK_BLOCK_LOG keys (or all N of them when N is smaller) of the
// blockIdx.y-th key array: size_lo == 2: every merge size 2 .. block (the block comes out sorted, direction by its global
// position); otherwise: the strides below the block size of the one merge of `size_lo` keys.
static __global__ void __launch_bounds__(512) lk_bitonic_block_kernel(fe *keys, uint64_t N, uint64_t size_lo, uint32_t full) {
    extern __shared__ uint4 lk_sm[];
    fe *sh = reinterpret_cast<fe *>(lk_sm);
    keys += blockIdx.y * N;
    const uint32_t BL = (uint32_t)(N < (1ull << H2_LK_BLOCK_LOG) ? N : (1ull << H2_LK_BLOCK_LOG));
    const uint64_t base = (uint64_t)blockIdx.x * BL;
    for (uint32_t e = threadIdx.x; e < BL; e += blockDim.x) sh[e] = fe_load(keys + base + e);
    __syncthreads();
    for (uint64_t size = full ? 2 : size_lo; size <= (full ? BL : size_lo); size <<= 1) {
        for (uint32_t stride = (uint32_t)(size / 2 < BL / 2 ? size / 2 : BL / 2); stride >= 1; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < BL / 2; t += blockDim.x) {
                const uint32_t i = (t / stride) * 2 * stride + (t % stride), j = i + stride;
                fe a = sh[i], b = sh[j];
                const bool asc = ((base + i) & size) == 0;
                bool lt = false;
#pragma unroll
                for (int k = 7; k >= 0; k--) if (a.v[k] != b.v[k]) { lt = b.v[k] < a.v[k]; break; }
                if (lt == asc) { sh[i] = b; sh[j] = a; }
            }
            __syncthreads();
        }
    }
    for (uint32_t e = threadIdx.x; e < BL; e += blockDim.x) fe_store(keys + base + e, sh[e]);
}
template <class P> __global__ void __launch_bounds__(256) lk_bitonic_global_kernel(fe *keys, uint64_t N, uint64_t size, uint64_t stride) {
    LookupPermute<P>::global_stage_body(keys + blockIdx.y * N, N, size, stride, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
// rank of every input row, histogram cnt (one atomic per distinct rank per warp), err = the lowest lookup with a miss
template <class P> __global__ void __launch_bounds__(128) lk_rank_kernel(LkCols c, const fe *keys, uint64_t N, uint64_t u, uint32_t *sc, uint32_t *err) {
    const uint64_t b = blockIdx.y, i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t r = H2_LK_NONE;
    bool miss = false;
    if (i < u) {
        r = LookupPermute<P>::rank_body(c.in[b], keys + b * N, u, i);
        miss = r == H2_LK_NONE;
    }
    if (miss) atomicMin(err, (uint32_t)b);
    const uint32_t peers = __match_any_sync(0xffffffffu, r);
    if (r != H2_LK_NONE && (threadIdx.x & 31) == (uint32_t)(__ffs(peers) - 1)) atomicAdd(sc + b * (u + 1) + r, (uint32_t)__popc(peers));
}
static __global__ void __launch_bounds__(256) lk_unconsumed_kernel(uint32_t *sc, uint64_t u, uint32_t count) {
    const uint64_t w = u + 1, b = blockIdx.y;
    lk_unconsumed_body(sc + b * w, u, sc + (count + b) * w, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
static __global__ void __launch_bounds__(256) lk_leftover_kernel(const uint32_t *sc, uint64_t u, uint32_t count, uint32_t *left) {
    const uint64_t w = u + 1, b = blockIdx.y;
    lk_leftover_body(sc + (count + b) * w, u, left + b * u, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
// rows [0, u) of both outputs, then with c.blind the blinding rows [u, u + rows); nothing when any lookup missed
template <class P> __global__ void __launch_bounds__(256) lk_fill_kernel(LkCols c, const fe *keys, uint64_t N, uint64_t u, uint64_t rows, const uint32_t *sc,
                                                                         uint32_t count, const uint32_t *left, const uint32_t *err) {
    if (*err != H2_LK_NONE) return;
    const uint64_t w = u + 1, b = blockIdx.y, i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < u) LookupPermute<P>::rank_fill_body(keys + b * N, u, sc + b * w, sc + (count + b) * w, left + b * u, c.out_in[b], c.out_tab[b], i);
    else if (c.blind) LookupPermute<P>::blind_body(c.blind + b * 2 * rows, rows, u, c.out_in[b], c.out_tab[b], i - u);
}
#endif

}  // namespace h2
