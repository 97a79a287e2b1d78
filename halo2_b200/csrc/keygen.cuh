// K19: the permutation argument's sigma polynomials from the copy-constraint mapping, resident.
//
//   build_vk / build_pk    /root/reference/halo2_proofs/src/plonk/permutation/keygen.rs:102-211
//                          sigma_i[j] = deltaomega[c][r] = delta^c * omega^r for (c, r) = mapping[i][j]
//
// The reference computes omega^0 .. omega^(n-1) with n serial multiplies, copies that row once per column times delta^c
// (cols x n products) and gathers from it.  Here nothing of size n is built: omega^r = hi[r >> h] * lo[r & (2^h - 1)] with
// lo[t] = omega^t (t < 2^h), hi[t] = (omega^(2^h))^t (t < 2^(k-h)), h = ceil(k / 2), and a table of delta^c (c < cols).
// Every table entry is its own square-and-multiply (no serial chain), and every sigma element is two multiplies of table
// entries that stay in L1 / L2: the pass is bound by reading 8 B of mapping and writing 32 B of result per element.
// Exact field arithmetic, so the bytes are THE elements the reference computes.
#pragma once
#include "field.cuh"

namespace h2 {

template <class P> struct KeygenOps {
    static H2_HD uint32_t split(uint32_t k) { return (k + 1) / 2; }
    static H2_HD uint64_t table_len(uint32_t k, uint32_t cols) { return (1ull << split(k)) + (1ull << (k - split(k))) + cols; }
    static H2_HD fe pow_u32(fe base, uint32_t e) {
        fe r = fe_one<P>();
        while (e) {
            if (e & 1) r = fe_mul<P>(r, base);
            e >>= 1;
            if (e) base = fe_sqr<P>(base);
        }
        return r;
    }
    // entry t of [lo (2^h) | hi (2^(k-h)) | delta^c (cols)]; omega, delta in Montgomery form
    static H2_HD void tables_body(fe *tab, const fe &omega, const fe &delta, uint32_t k, uint32_t cols, uint64_t t) {
        const uint32_t h = split(k);
        const uint64_t nlo = 1ull << h, nhi = 1ull << (k - h);
        if (t >= nlo + nhi + cols) return;
        fe base;
        uint32_t e;
        if (t < nlo) { base = omega; e = (uint32_t)t; }
        else if (t < nlo + nhi) {
            base = omega;
            for (uint32_t s = 0; s < h; s++) base = fe_sqr<P>(base);   // omega^(2^h)
            e = (uint32_t)(t - nlo);
        } else { base = delta; e = (uint32_t)(t - nlo - nhi); }
        fe_store(tab + t, pow_u32(base, e));
    }
    // dst[t] = delta^c * omega^r for (c, r) = map[t], t < count; returns 1 (and writes nothing) for an entry outside (cols, 2^k)
    static H2_HD uint32_t sigma_body(fe *dst, const uint2 *map, const fe *tab, uint32_t k, uint32_t cols, uint64_t count, uint64_t t) {
        if (t >= count) return 0;
        const uint2 cr = map[t];
        if (cr.x >= cols || (uint64_t)cr.y >= (1ull << k)) return 1;
        const uint32_t h = split(k);
        const fe *lo = tab, *hi = tab + (1ull << h), *dpow = hi + (1ull << (k - h));
        const fe w = fe_mul<P>(fe_load(hi + (cr.y >> h)), fe_load(lo + (cr.y & ((1u << h) - 1))));
        fe_store(dst + t, fe_mul<P>(fe_load(dpow + cr.x), w));
        return 0;
    }
};

#if defined(__CUDACC__)
template <class P> __global__ void __launch_bounds__(128) keygen_tables_kernel(fe *tab, fe omega, fe delta, uint32_t k, uint32_t cols) {
    KeygenOps<P>::tables_body(tab, omega, delta, k, cols, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P>
__global__ void __launch_bounds__(256) keygen_sigma_kernel(fe *dst, const uint2 *map, const fe *tab, uint32_t k, uint32_t cols, uint64_t count, uint32_t *err) {
    if (KeygenOps<P>::sigma_body(dst, map, tab, k, cols, count, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x)) *err = 1;
}
#endif

}  // namespace h2
