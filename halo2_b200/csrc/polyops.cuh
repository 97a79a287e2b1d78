// K14: the prover's coefficient-form reductions on resident polynomials -- SURVEY.md section 8(f) row 3.
//
//   eval_polynomial        /root/reference/halo2_proofs/src/arithmetic.rs:297-303   sum_i a_i x^i (Horner in the reference)
//   compute_inner_product  arithmetic.rs:308-319                                     sum_i a_i b_i
//   kate_division          arithmetic.rs:322-341                                     q = (a - a(b)) / (X - b):  q_i = sum_{j>i} a_j b^(j-i-1)
//   divide_by_vanishing_poly  poly/domain.rs:329-348                                  h_i *= 1 / t(zeta w^i), elementwise over the extended domain
//
// The reference runs all three serially ("TODO: parallelize?"); each is a first-order linear recurrence, so each becomes a
// tree of CHUNK-sized serial pieces: level l turns m values into ceil(m / CHUNK) by CHUNK multiply-adds per thread with the
// point raised to CHUNK^l.  k = 14: 16384 -> 512 -> 16 -> 1, three launches of 32 dependent multiplies instead of 16384.
// Exact field arithmetic: the result is THE field element the reference computes, whatever the association order.
//
// Layout: `batch` polynomials of `n` coefficients (Montgomery form, device pointers in an array -- the buffers of h2_poly_*
// handles), one point per polynomial; partial levels live in one scratch array [batch][m].
#pragma once
#include "field.cuh"

namespace h2 {

#define H2_POLY_CHUNK 32

// The levels of a chunk tree over `batch` columns of n values: level 0 is the caller's data, level l = 1 ... L lives in
// scratch at off[l] as [batch][m[l]], m[l + 1] = ceil(m[l] / CHUNK).  Kernels that walk the levels themselves take the
// GpLevels part by value (gp_carry_kernel).  A reduction of n < 2^32 values takes all 8 entries: 2^32 - 1, 2^27, ..., 4, 1.
#define H2_GP_MAX_LEVELS 8
struct GpLevels {
    uint64_t m[H2_GP_MAX_LEVELS], off[H2_GP_MAX_LEVELS];
    uint32_t L;
};
// The plan of one call: its levels and the elements they take in each level array (po_lvl, po_q).  The plans below return
// nullptr, or the reason n is refused.
struct GpTree : GpLevels {
    uint64_t total;
};
constexpr const char *gp_push_level(GpTree *T, uint64_t batch) {
    if (T->L + 1 >= H2_GP_MAX_LEVELS) return "n needs more chunk-tree levels than H2_GP_MAX_LEVELS";
    T->off[T->L + 1] = T->L ? T->off[T->L] + T->m[T->L] * batch : 0;
    T->m[T->L + 1] = (T->m[T->L] + H2_POLY_CHUNK - 1) / H2_POLY_CHUNK;
    T->L++;
    T->total = T->off[T->L] + T->m[T->L] * batch;
    return nullptr;
}
// The reduction to one value (eval, inner product, kate division).  `inner`: a length-1 inner product still gets its
// product level.
constexpr const char *gp_reduce_plan(uint64_t n, uint64_t batch, bool inner, GpTree *T) {
    *T = GpTree{};
    T->m[0] = n;
    while (T->m[T->L] > 1)
        if (const char *e = gp_push_level(T, batch)) return e;
    if (inner && T->L == 0) { T->m[1] = 1; T->L = 1; T->total = batch; }
    return nullptr;
}
// The scan down to <= CHUNK values (the running product, K21's product columns).  `level1`: level 1 even when n <= CHUNK.
constexpr const char *gp_scan_plan(uint64_t n, uint64_t batch, bool level1, GpTree *T) {
    *T = GpTree{};
    T->m[0] = n;
    while (T->m[T->L] > H2_POLY_CHUNK || (level1 && T->L == 0))
        if (const char *e = gp_push_level(T, batch)) return e;
    return nullptr;
}
static_assert([] { GpTree T{}; return !gp_reduce_plan(0xFFFFFFFFull, 1, false, &T) && T.L + 1 == H2_GP_MAX_LEVELS; }(),
              "a reduction of n < 2^32 values fits GpLevels");

template <class P> struct PolyOps {
    // level of eval_polynomial: out[b][t] = sum_{i < CHUNK} in_b[t CHUNK + i] x_b^i   (Horner from the top of the chunk)
    // in_ptrs != nullptr: level 0 reads polynomial b from in_ptrs[b]; else from in_flat + b * m
    static H2_HD void eval_level_body(const fe *const *in_ptrs, const fe *in_flat, uint64_t m, const fe *points, fe *out, uint64_t out_m, uint32_t b,
                                      uint64_t t) {
        if (t >= out_m) return;
        const fe *src = in_ptrs ? in_ptrs[b] : in_flat + (uint64_t)b * m;
        const fe x = fe_load(points + b);
        const uint64_t lo = t * H2_POLY_CHUNK, hi = lo + H2_POLY_CHUNK < m ? lo + H2_POLY_CHUNK : m;
        fe acc = fe_zero();
        for (uint64_t i = hi; i-- > lo;) acc = fe_add<P>(fe_mul<P>(acc, x), fe_load(src + i));
        fe_store(out + (uint64_t)b * out_m + t, acc);
    }
    // points_out[b] = points_in[b]^CHUNK (CHUNK = 2^5)
    static H2_HD void pow_chunk_body(const fe *in, fe *out, uint32_t b) {
        fe x = fe_load(in + b);
        for (uint32_t c = H2_POLY_CHUNK; c > 1; c >>= 1) x = fe_sqr<P>(x);
        fe_store(out + b, x);
    }
    // level 0 of compute_inner_product: out[b][t] = sum_{i in chunk t} a_b[i] * c_b[i]; the upper levels are eval levels at x = 1
    static H2_HD void inner_level0_body(const fe *const *a_ptrs, const fe *const *c_ptrs, uint64_t m, fe *out, uint64_t out_m, uint32_t b, uint64_t t) {
        if (t >= out_m) return;
        const fe *a = a_ptrs[b], *c = c_ptrs[b];
        const uint64_t lo = t * H2_POLY_CHUNK, hi = lo + H2_POLY_CHUNK < m ? lo + H2_POLY_CHUNK : m;
        fe acc = fe_zero();
        for (uint64_t i = lo; i < hi; i++) acc = fe_add<P>(acc, fe_mul<P>(fe_load(a + i), fe_load(c + i)));
        fe_store(out + (uint64_t)b * out_m + t, acc);
    }
    // kate_division, downward pass of one level.  With Q(i) = sum_{j >= i} a_j x^(j-i) (so q_i = Q(i + 1)) a chunk [lo, hi)
    // satisfies Q(lo) = V + x^len Q(hi), V = the chunk's eval-level value: the upward pass IS the eval tree.  Going down,
    // thread t of a level takes the carry Q(hi) from the level above (carry_in[b][t + 1], zero past the end) and walks its chunk
    // from the top, writing Q at every position of the level below (or, at level 0, q_i = Q(i + 1) into the quotient).
    //   vals: the level's own values [b][m] (level 0: the polynomial, via in_ptrs);  carry_in: Q at the chunk boundaries of this
    //   level = the level above's Q array [b][out_m] (nullptr at the top level: no carry);  q_out: level 0 only.
    static H2_HD void kate_down_body(const fe *const *in_ptrs, const fe *in_flat, uint64_t m, const fe *points, const fe *carry_in, uint64_t out_m,
                                     fe *q_below, fe *const *q_out_ptrs, uint32_t b, uint64_t t) {
        if (t >= out_m) return;
        const fe *src = in_ptrs ? in_ptrs[b] : in_flat + (uint64_t)b * m;
        const fe x = fe_load(points + b);
        const uint64_t lo = t * H2_POLY_CHUNK, hi = lo + H2_POLY_CHUNK < m ? lo + H2_POLY_CHUNK : m;
        fe acc = (carry_in && t + 1 < out_m) ? fe_load(carry_in + (uint64_t)b * out_m + t + 1) : fe_zero();   // Q(hi)
        for (uint64_t i = hi; i-- > lo;) {
            acc = fe_add<P>(fe_mul<P>(acc, x), fe_load(src + i));      // Q(i)
            if (q_out_ptrs) { if (i >= 1) fe_store(q_out_ptrs[b] + (i - 1), acc); }   // q_(i-1) = Q(i); Q(0) = a(x) is dropped
            else fe_store(q_below + (uint64_t)b * m + i, acc);
        }
    }
};

// The permutation argument's grand product (plonk/permutation/prover.rs:98-157; the lookup argument has the same shape,
// plonk/lookup/prover.rs): `modified_values.batch_invert()` and the running product z[0] = last_z, z[i] = z[i-1] * mv[i-1].
template <class P> struct GrandProduct {
    // ff::BatchInvert in place: a[i] <- 1 / a[i], zeros stay zero.  Thread t owns 16 elements, one inversion (Montgomery's trick).
    static H2_HD void invert_body(fe *a, uint64_t n, uint64_t t) {
        const uint64_t lo = t * 16;
        if (lo >= n) return;
        const uint32_t m = (uint32_t)(n - lo < 16 ? n - lo : 16);
        fe pre[16], v[16];
        fe acc = fe_one<P>();
        for (uint32_t i = 0; i < m; i++) {
            v[i] = fe_load(a + lo + i);
            pre[i] = acc;
            if (!fe_is_zero(v[i])) acc = fe_mul<P>(acc, v[i]);
        }
        acc = fe_inv_gcd<P>(acc);
        for (uint32_t i = m; i-- > 0;) {
            if (fe_is_zero(v[i])) continue;
            fe_store(a + lo + i, fe_mul<P>(acc, pre[i]));
            acc = fe_mul<P>(acc, v[i]);
        }
    }
    // upward level of the running product: out[t] = prod of chunk t of in (m values)
    static H2_HD void up_body(const fe *in, uint64_t m, fe *out, uint64_t out_m, uint64_t t) {
        if (t >= out_m) return;
        const uint64_t lo = t * H2_POLY_CHUNK, hi = lo + H2_POLY_CHUNK < m ? lo + H2_POLY_CHUNK : m;
        fe acc = fe_load(in + lo);
        for (uint64_t i = lo + 1; i < hi; i++) acc = fe_mul<P>(acc, fe_load(in + i));
        fe_store(out + t, acc);
    }
    // downward level: E[i] = carry_t * prod_{lo <= j < i} in[j] for i in chunk t (the exclusive running product), with
    // carry_t = E_above[t] (or `init` at the top level, where there is one chunk).  `count` positions are written (level 0 writes
    // n outputs from n - 1... inputs: the last input is never used, plonk/permutation/prover.rs:150-156).
    static H2_HD void down_body(const fe *in, uint64_t m, const fe *carry_above, const fe &init, fe *out, uint64_t out_m, uint64_t t) {
        if (t >= out_m) return;
        const uint64_t lo = t * H2_POLY_CHUNK, hi = lo + H2_POLY_CHUNK < m ? lo + H2_POLY_CHUNK : m;
        fe acc = carry_above ? fe_load(carry_above + t) : init;
        for (uint64_t i = lo; i < hi; i++) {
            fe_store(out + i, acc);
            acc = fe_mul<P>(acc, fe_load(in + i));
        }
    }
};

// divide_by_vanishing_poly (poly/domain.rs:329-348): h[i] *= t_evaluations[i mod len], len = 2^(extended_k - k) inverses of
// t(X) = X^n - 1 over the coset (domain.rs:86-128), Montgomery form
template <class P> struct VanishDiv {
    static H2_HD void body(fe *a, uint64_t n, const fe *t, uint32_t t_mask, uint64_t i) {
        if (i < n) fe_store(a + i, fe_mul<P>(fe_load(a + i), fe_load(t + (i & t_mask))));
    }
};

#if defined(__CUDACC__)
template <class P> __global__ void __launch_bounds__(64) poly_batch_invert_kernel(fe *a, uint64_t n) {
    GrandProduct<P>::invert_body(a, n, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P> __global__ void __launch_bounds__(128) poly_product_up_kernel(const fe *in, uint64_t m, fe *out, uint64_t out_m) {
    GrandProduct<P>::up_body(in, m, out, out_m, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P> __global__ void __launch_bounds__(128) poly_product_down_kernel(const fe *in, uint64_t m, const fe *carry_above, fe init, fe *out,
                                                                                   uint64_t out_m) {
    GrandProduct<P>::down_body(in, m, carry_above, init, out, out_m, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P> __global__ void __launch_bounds__(256) poly_vanish_div_kernel(fe *a, uint64_t n, const fe *t, uint32_t t_mask) {
    VanishDiv<P>::body(a, n, t, t_mask, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P> __global__ void __launch_bounds__(128) poly_eval_level_kernel(const fe *const *in_ptrs, const fe *in_flat, uint64_t m, const fe *points,
                                                                                 fe *out, uint64_t out_m) {
    PolyOps<P>::eval_level_body(in_ptrs, in_flat, m, points, out, out_m, blockIdx.y, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
// Small polynomials (n <= 2^16: every k <= 16 column) in ONE launch, one CTA per polynomial: thread t runs Horner over its
// own slice of ceil(n / 1024) coefficients, then the 1024 slice values combine in a shared-memory tree, v_t += x^(len 2^l)
// v_(t + 2^l): ~16 + 10 dependent multiply-adds instead of three levels of launches.  OPT-IN (h2_test_set_poly_cta): one CTA's
// serial slices leave most SMs idle where the level tree fills the machine (ctx.cuh).  Same field element as the serial loop -- exact arithmetic.
#define H2_POLY_CTA 1024
template <class P> __device__ __forceinline__ fe poly_pow_small(fe x, uint32_t e) {      // x^e, e >= 1 small
    fe r = x;
    uint32_t top = 31 - __clz(e);
    for (int b = (int)top - 1; b >= 0; b--) { r = fe_sqr<P>(r); if ((e >> b) & 1u) r = fe_mul<P>(r, x); }
    return r;
}
template <class P> __global__ void __launch_bounds__(H2_POLY_CTA) poly_eval_cta_kernel(const fe *const *polys, uint64_t n, const fe *points, fe *out) {
    __shared__ fe sh[H2_POLY_CTA];
    const uint32_t b = blockIdx.x, t = threadIdx.x;
    const fe *a = polys[b];
    const fe x = fe_load(points + b);
    const uint32_t per = (uint32_t)((n + H2_POLY_CTA - 1) / H2_POLY_CTA);
    const uint64_t lo = (uint64_t)t * per, hi = lo + per < n ? lo + per : n;
    fe acc = fe_zero();
    for (uint64_t i = hi; i > lo; i--) acc = fe_add<P>(fe_mul<P>(acc, x), fe_load(a + i - 1));
    sh[t] = acc;
    fe xp = poly_pow_small<P>(x, per);                   // x^per: the weight of the right neighbour
    __syncthreads();
    for (uint32_t stride = 1; stride < H2_POLY_CTA; stride <<= 1) {
        if ((t & (2 * stride - 1)) == 0) sh[t] = fe_add<P>(sh[t], fe_mul<P>(xp, sh[t + stride]));
        xp = fe_sqr<P>(xp);
        __syncthreads();
    }
    if (t == 0) fe_store(out + b, sh[0]);
}
// kate_division the same way: with Q(i) = sum_{j >= i} a_j x^(j - i) (q_i = Q(i + 1)) a slice [lo, hi) has
// Q(lo) = V + x^len Q(hi).  Thread t computes its slice value V_t, a shared-memory suffix scan of the affine maps
// (V, x^len) -- (V1, p1) o (V2, p2) = (V1 + p1 V2, p1 p2), 10 steps -- gives every slice its carry Q(hi), and a second walk
// over the slice writes the quotient.  The n - 1 quotient coefficients go to dst; slot n - 1 is cleared by the caller.
#define H2_KATE_CTA 512      // two 32-byte arrays of the scan: 32 KiB of static shared memory
template <class P> __global__ void __launch_bounds__(H2_KATE_CTA) poly_kate_cta_kernel(const fe *const *polys, uint64_t n, const fe *points, fe *const *dst) {
    __shared__ fe sv[H2_KATE_CTA], sp[H2_KATE_CTA];
    const uint32_t b = blockIdx.x, t = threadIdx.x;
    const fe *a = polys[b];
    fe *q = dst[b];
    const fe x = fe_load(points + b);
    const uint32_t per = (uint32_t)((n + H2_KATE_CTA - 1) / H2_KATE_CTA);
    const uint64_t lo = (uint64_t)t * per < n ? (uint64_t)t * per : n, hi = lo + per < n ? lo + per : n;
    fe acc = fe_zero();
    for (uint64_t i = hi; i > lo; i--) acc = fe_add<P>(fe_mul<P>(acc, x), fe_load(a + i - 1));
    // the map of this slice: Q(lo) = V + p Q(hi), p = x^(hi - lo) (an empty slice is the identity map (0, 1))
    fe v = acc, pw = hi > lo ? poly_pow_small<P>(x, (uint32_t)(hi - lo)) : fe_one<P>();
    sv[t] = v; sp[t] = pw;
    __syncthreads();
    // inclusive suffix scan: after it (sv[t], sp[t]) maps Q(n) = 0 ... to Q(lo_t), i.e. sv[t] = Q(lo_t)
    for (uint32_t stride = 1; stride < H2_KATE_CTA; stride <<= 1) {
        fe v2 = fe_zero(), p2 = fe_one<P>();
        const bool has = t + stride < H2_KATE_CTA;
        if (has) { v2 = sv[t + stride]; p2 = sp[t + stride]; }
        __syncthreads();
        if (has) { v = fe_add<P>(v, fe_mul<P>(pw, v2)); pw = fe_mul<P>(pw, p2); sv[t] = v; sp[t] = pw; }
        __syncthreads();
    }
    // carry of this slice = Q(hi_t) = Q(lo_(t+1)) (0 past the end); walk down writing q_(i-1) = Q(i)
    fe carry = (t + 1 < H2_KATE_CTA) ? sv[t + 1] : fe_zero();
    for (uint64_t i = hi; i > lo; i--) {
        carry = fe_add<P>(fe_mul<P>(carry, x), fe_load(a + i - 1));   // Q(i - 1)
        if (i - 1 >= 1) fe_store(q + (i - 2), carry);                 // q_(i-2) = Q(i - 1); Q(0) = a(x) is dropped
    }
}
template <class P> __global__ void poly_pow_chunk_kernel(const fe *in, fe *out, uint32_t batch) {
    uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < batch) PolyOps<P>::pow_chunk_body(in, out, b);
}
template <class P> __global__ void __launch_bounds__(128) poly_inner_level0_kernel(const fe *const *a_ptrs, const fe *const *c_ptrs, uint64_t m, fe *out,
                                                                                   uint64_t out_m) {
    PolyOps<P>::inner_level0_body(a_ptrs, c_ptrs, m, out, out_m, blockIdx.y, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P> __global__ void __launch_bounds__(128) poly_kate_down_kernel(const fe *const *in_ptrs, const fe *in_flat, uint64_t m, const fe *points,
                                                                                const fe *carry_in, uint64_t out_m, fe *q_below, fe *const *q_out_ptrs) {
    PolyOps<P>::kate_down_body(in_ptrs, in_flat, m, points, carry_in, out_m, q_below, q_out_ptrs, blockIdx.y,
                               (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
template <class P> __global__ void fe_fill_kernel(fe *a, uint32_t n, fe v) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fe_store(a + i, v);
}
#endif

}  // namespace h2
