// K21: the permutation and lookup arguments' product columns, every set of every proof in one call.
//
//   permutation::Argument::commit   /root/reference/halo2_proofs/src/plonk/permutation/prover.rs:98-168
//   lookup::Permuted::commit_product                     plonk/lookup/prover.rs:279-337
//
// Row b of the batch (grid.y) is one product column: (proof, set) of the permutation, or (proof, lookup).
//   1. factors   den_b[i] -> scratch, num_b[i] -> z_b (the output doubles as the numerators' buffer):
//        permutation  den = prod_j (v_j[i] + beta sigma_j[i] + gamma),  num = prod_j (v_j[i] + beta delta^(c0+j) omega^i + gamma)
//                     (c0 + j = the column's position in the argument's column list; omega^i = hi[i >> h] * lo[i & mask] and
//                     delta^c from K19's tables -- nothing of size n is built)
//        lookup       den = (beta + a'[i]) (gamma + s'[i]),  num = (a[i] + beta) (s[i] + gamma)
//   2. ff::BatchInvert of every den (K14's Montgomery-trick body over the flat scratch: zeros stay zero).
//   3. level 0 of the running product: mv = num * den^-1 back into the scratch, and the chunk products -- K14's chunk tree
//      (GrandProduct::up_body / down_body) batched over grid.y, every column from 1.
//   4. carries: a column's z[n - bf - 1] from 1 is its exclusive prefix product at p = n - bf - 1, which the upward tree
//      already holds -- the products of the chunks before p's chunk at every level, <= 31 per level.  A proof's chain starts
//      at ONE and c_(a+1) = c_a * z'_a[p] (the reference's last_z hand-over, permutation/prover.rs:81, :163); a lookup is a
//      chain of one column, so its carry is 1 (z[0] = ONE, lookup/prover.rs:310-315).
//   5. the downward pass of the tree starts each column at its carry and writes z_b; then the bf caller values go into rows
//      [n - bf, n) (:155-161 / :317-321).
// Exact field arithmetic, so z equals the reference's serial loop element for element: z_a = c_a * z'_a on every row below
// n - bf, and row n - bf - 1, the one that carries, is never a blinding row.
#pragma once
#include "polyops.cuh"
#include "keygen.cuh"

namespace h2 {

// The product columns' chunk tree is gp_scan_plan's with level 1 always present (polyops.cuh); its level 0 is the flat
// [batch][n] scratch of step 3.

template <class P> struct ProductArgs {
    // permutation factors of row i of column b = (proof, set) = (b / sets, b % sets); cols: proofs x ncols column pointers
    static H2_HD void perm_factors_body(const fe *const *cols, const fe *const *sigmas, uint32_t ncols, uint32_t chunk_len, uint32_t sets,
                                        const fe *tab, uint32_t k, const fe &beta, const fe &gamma, fe *den, fe *const *z, uint32_t b,
                                        uint64_t i) {
        const uint64_t n = 1ull << k;
        if (i >= n) return;
        const uint32_t proof = b / sets, c0 = (b % sets) * chunk_len;
        const uint32_t len = ncols - c0 < chunk_len ? ncols - c0 : chunk_len;
        const uint32_t h = KeygenOps<P>::split(k);
        const fe *lo = tab, *hi = tab + (1ull << h), *dpow = hi + (1ull << (k - h));
        const fe bw = fe_mul<P>(beta, fe_mul<P>(fe_load(hi + (i >> h)), fe_load(lo + (i & ((1ull << h) - 1)))));   // beta omega^i
        fe d = fe_one<P>(), u = fe_one<P>();
        for (uint32_t j = 0; j < len; j++) {
            const fe v = fe_add<P>(fe_load(cols[(uint64_t)proof * ncols + c0 + j] + i), gamma);
            d = fe_mul<P>(d, fe_add<P>(v, fe_mul<P>(beta, fe_load(sigmas[c0 + j] + i))));
            u = fe_mul<P>(u, fe_add<P>(v, fe_mul<P>(bw, fe_load(dpow + c0 + j))));
        }
        fe_store(den + (uint64_t)b * n + i, d);
        fe_store(z[b] + i, u);
    }
    // lookup factors of row i of column b; io: per column b its (input, table, permuted input, permuted table)
    static H2_HD void lookup_factors_body(const fe *const *io, uint64_t n, const fe &beta, const fe &gamma, fe *den, fe *const *z, uint32_t b,
                                          uint64_t i) {
        if (i >= n) return;
        const fe *const *c = io + 4ull * b;
        fe_store(den + (uint64_t)b * n + i, fe_mul<P>(fe_add<P>(beta, fe_load(c[2] + i)), fe_add<P>(gamma, fe_load(c[3] + i))));
        fe_store(z[b] + i, fe_mul<P>(fe_add<P>(fe_load(c[0] + i), beta), fe_add<P>(fe_load(c[1] + i), gamma)));
    }
    // level 0 of the upward tree with the numerators folded in: mv = num * den^-1 replaces den^-1, out[b][t] = product of chunk t
    static H2_HD void mv_up_body(const fe *const *z, fe *mv, uint64_t n, fe *out, uint64_t out_m, uint32_t b, uint64_t t) {
        if (t >= out_m) return;
        const uint64_t lo = t * H2_POLY_CHUNK, hi = lo + H2_POLY_CHUNK < n ? lo + H2_POLY_CHUNK : n;
        const fe *num = z[b];
        fe *a = mv + (uint64_t)b * n;
        fe acc = fe_one<P>();
        for (uint64_t i = lo; i < hi; i++) {
            const fe x = fe_mul<P>(fe_load(num + i), fe_load(a + i));
            fe_store(a + i, x);
            acc = fe_mul<P>(acc, x);
        }
        fe_store(out + (uint64_t)b * out_m + t, acc);
    }
    // the carries of one proof's chain of `sets` columns: init[b] = c_a for b = proof * sets + a
    static H2_HD void carry_body(const fe *mv, const fe *lvl, const GpLevels &G, uint64_t p, uint32_t sets, fe *init, uint32_t proof) {
        fe c = fe_one<P>();
        for (uint32_t a = 0; a < sets; a++) {
            const uint64_t b = (uint64_t)proof * sets + a;
            fe_store(init + b, c);
            if (a + 1 == sets) break;
            for (uint32_t l = 0; l <= G.L; l++) {                    // z'[p] = prod over levels of the chunks before p's, within its parent
                const uint64_t pl = p >> (5 * l);
                const fe *v = l == 0 ? mv + b * G.m[0] : lvl + G.off[l] + b * G.m[l];
                for (uint64_t j = pl & ~(uint64_t)(H2_POLY_CHUNK - 1); j < pl; j++) c = fe_mul<P>(c, fe_load(v + j));
            }
        }
    }
    // the caller's blinding values: z_b[n - bf + r] = blind[b * bf + r]
    static H2_HD void blind_body(fe *const *z, uint64_t n, uint32_t bf, const fe *blind, uint64_t count, uint64_t idx) {
        if (idx >= count * bf) return;
        const uint64_t b = idx / bf, r = idx % bf;
        fe_store(z[b] + (n - bf + r), fe_load(blind + idx));
    }
};
static_assert(H2_POLY_CHUNK == 32, "carry_body steps levels by 5 bits");

#if defined(__CUDACC__)
template <class P>
__global__ void __launch_bounds__(128) gp_perm_factors_kernel(const fe *const *cols, const fe *const *sigmas, uint32_t ncols, uint32_t chunk_len,
                                                              uint32_t sets, const fe *tab, uint32_t k, fe beta, fe gamma, fe *den, fe *const *z) {
    ProductArgs<P>::perm_factors_body(cols, sigmas, ncols, chunk_len, sets, tab, k, beta, gamma, den, z, blockIdx.y,
                                      (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P>
__global__ void __launch_bounds__(256) gp_lookup_factors_kernel(const fe *const *io, uint64_t n, fe beta, fe gamma, fe *den, fe *const *z) {
    ProductArgs<P>::lookup_factors_body(io, n, beta, gamma, den, z, blockIdx.y, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P> __global__ void __launch_bounds__(128) gp_mv_up_kernel(const fe *const *z, fe *mv, uint64_t n, fe *out, uint64_t out_m) {
    ProductArgs<P>::mv_up_body(z, mv, n, out, out_m, blockIdx.y, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
// K14's upward / downward levels, column blockIdx.y of the flat [batch][m] arrays
template <class P> __global__ void __launch_bounds__(128) gp_up_kernel(const fe *in, uint64_t m, fe *out, uint64_t out_m) {
    const uint64_t b = blockIdx.y;
    GrandProduct<P>::up_body(in + b * m, m, out + b * out_m, out_m, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P>
__global__ void __launch_bounds__(128) gp_down_kernel(const fe *in, uint64_t m, const fe *carry_above, const fe *init, fe *out, fe *const *z,
                                                      uint64_t out_m) {
    const uint64_t b = blockIdx.y;
    GrandProduct<P>::down_body(in + b * m, m, carry_above ? carry_above + b * out_m : nullptr, fe_load(init + b), z ? z[b] : out + b * m, out_m,
                               (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P> __global__ void gp_carry_kernel(const fe *mv, const fe *lvl, GpLevels G, uint64_t p, uint32_t sets, fe *init, uint32_t proofs) {
    const uint32_t proof = blockIdx.x * blockDim.x + threadIdx.x;
    if (proof < proofs) ProductArgs<P>::carry_body(mv, lvl, G, p, sets, init, proof);
}
template <class P> __global__ void __launch_bounds__(256) gp_blind_kernel(fe *const *z, uint64_t n, uint32_t bf, const fe *blind, uint64_t count) {
    ProductArgs<P>::blind_body(z, n, bf, blind, count, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
#endif

}  // namespace h2
