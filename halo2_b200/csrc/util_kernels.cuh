// Small kernels several translation units launch: representation conversions, seeded generators, self-test and
// microbenchmark kernels, the G-term point sum.
#pragma once
#include "ctx.cuh"
#include "msm.cuh"   // ld_affine / st_affine, xyzz helpers
#include "ecfft.cuh" // the EC-FFT's warp-uniform group law (self-test kernel)

// ------------------------------------------------------------------------------------------------
// small kernels: conversions, generators, self-tests
// ------------------------------------------------------------------------------------------------
template <class P> __global__ void convert_kernel(fe *a, uint64_t n, int to_mont) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe x = fe_load(a + i);
    fe_store(a + i, to_mont ? fe_to_mont<P>(x) : fe_from_mont<P>(x));
}
// affine points: identity (0,0) maps to itself under both conversions
template <class P> __global__ void convert_points_kernel(affine *a, uint64_t n, int to_mont) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    affine p = ld_affine(a + i);
    if (to_mont) { p.x = fe_to_mont<P>(p.x); p.y = fe_to_mont<P>(p.y); }
    else { p.x = fe_from_mont<P>(p.x); p.y = fe_from_mont<P>(p.y); }
    st_affine(a + i, p);
}
template <class P> __device__ affine xyzz_to_affine_dev(const xyzz &p) {
    affine r;
    if (xyzz_is_identity(p)) { r.x = fe_zero(); r.y = fe_zero(); return r; }
    fe t = fe_inv_gcd<P>(fe_mul<P>(p.zz, p.zzz));
    r.x = fe_mul<P>(p.x, fe_mul<P>(t, p.zzz));   // X / ZZ
    r.y = fe_mul<P>(p.y, fe_mul<P>(t, p.zz));    // Y / ZZZ
    return r;
}
template <class P> __global__ void __launch_bounds__(128) gen_points_kernel(affine *out, uint64_t seed, uint64_t first, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t s = splitmix64(seed ^ splitmix64(first + i)) | 1ULL;
    affine g;
    g.x = fe_neg<P>(fe_one<P>());
    g.y = fe_dbl<P>(fe_one<P>());
    xyzz acc = xyzz_identity();
    for (int b = 63; b >= 0; b--) {
        xyzz_double<P>(acc);
        if ((s >> b) & 1ULL) xyzz_add_mixed<P>(acc, g);
    }
    st_affine(out + i, xyzz_to_affine_dev<P>(acc));
}
template <class P> __global__ void test_field_kernel(const fe *a, const fe *b, fe *out, uint64_t n, int op) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fe x = fe_to_mont<P>(fe_load(a + i)), y = fe_to_mont<P>(fe_load(b + i)), r;
    switch (op) {
    case 0: r = fe_add<P>(x, y); break;
    case 1: r = fe_sub<P>(x, y); break;
    case 2: r = fe_mul<P>(x, y); break;
    case 3: r = fe_inv<P>(x); break;
    case 5: r = fe_inv_gcd<P>(x); break;
    default: r = fe_sqr<P>(x); break;
    }
    fe_store(out + i, fe_from_mont<P>(r));
}
// Group-law self-tests (h2_test_curve_op; the ops are listed in include/halo2_b200.h).  Points arrive and leave as canonical
// affine points.  Ops 3 .. 13 rescale their XYZZ operands by test_lambda, so the formulas see ZZ != 1 (except on every 4th
// element); the result is compared as an affine point, which does not depend on the representation.
template <class P> __device__ void mont_point(affine &p) {
    if (!affine_is_identity(p)) { p.x = fe_to_mont<P>(p.x); p.y = fe_to_mont<P>(p.y); }
}
template <class P> __device__ void st_canonical(affine *out, affine o) {
    o.x = fe_from_mont<P>(o.x); o.y = fe_from_mont<P>(o.y);
    st_affine(out, o);
}
template <class P> __device__ affine poison_point() {   // (1, 0) canonical: not on the curve
    affine o; o.x = fe_one<P>(); o.y = fe_zero();
    return o;
}
template <class P> __global__ void __launch_bounds__(64) test_curve_kernel(const affine *a, const affine *b, affine *out, uint64_t n, int op) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    affine pa = ld_affine(a + i), pb = ld_affine(b + i);
    mont_point<P>(pa);
    xyzz r = xyzz_from_affine<P>(pa);
    if (op == 0) {
        mont_point<P>(pb);
        xyzz t = r;
        xyzz_add_mixed<P>(r, pb);                         // mixed path
        xyzz full = xyzz_from_affine<P>(pb);
        xyzz_add<P>(t, full);                             // full-add path must agree
        affine r1 = xyzz_to_affine_dev<P>(r), r2 = xyzz_to_affine_dev<P>(t);
        if (!(fe_eq(r1.x, r2.x) && fe_eq(r1.y, r2.y))) r1 = poison_point<P>();
        st_canonical<P>(out + i, r1);
        return;
    } else if (op == 1) {
        xyzz_double<P>(r);
    } else if (op == 2) {
        uint32_t k[8];
        for (int j = 0; j < 8; j++) k[j] = pb.x.v[j];
        r = xyzz_scalar_mul<P>(pa, k);
    } else {                                              // 3 .. 6: the serial forms on rescaled operands
        r = xyzz_rescale<P>(r, test_lambda<P>(i, 0));
        if (op == 6) xyzz_shift<P>(r, pb.x.v[0]);         // k = the low 32 bits of b.x
        else if (op == 5) xyzz_double<P>(r);
        else {
            mont_point<P>(pb);
            if (op == 4) xyzz_add_mixed<P>(r, pb);
            else xyzz_add<P>(r, xyzz_rescale<P>(xyzz_from_affine<P>(pb), test_lambda<P>(i, 1)));
        }
    }
    st_canonical<P>(out + i, xyzz_to_affine_dev<P>(r));
}
// Ops 7 .. 13: the lane-cooperative forms, `lanes` consecutive lanes per element (2 for the pair of op 9, 4 otherwise).  The
// launch is whole warps and nothing returns before the group law: lanes past n hold identity operands and still reach every
// shuffle, as xyzz_addsub_q / xyzz_double_q require of the full warp.  Every lane of a group computes the result; if any lane's
// XYZZ words differ from the group's first lane the element gets the poison point -- the forms rely on the lanes staying equal.
template <class P> __global__ void __launch_bounds__(64) test_curve_coop_kernel(const affine *a, const affine *b, affine *out, uint64_t n, int op) {
    const uint32_t lanes = op == 9 ? 2u : 4u;
    const uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / lanes;
    affine pa, pb;
    pa.x = pa.y = pb.x = pb.y = fe_zero();
    if (i < n) { pa = ld_affine(a + i); pb = ld_affine(b + i); }
    mont_point<P>(pa);
    const uint32_t k = pb.x.v[0];                         // op 10: the shift count, the low 32 bits of b.x
    if (op != 10) mont_point<P>(pb);
    xyzz r = xyzz_rescale<P>(xyzz_from_affine<P>(pa), test_lambda<P>(i, 0));
    const xyzz q = xyzz_rescale<P>(xyzz_from_affine<P>(pb), test_lambda<P>(i, 1));
    switch (op) {
    case 7: xyzz_add_quad<P>(r, q); break;
    case 8: xyzz_add_mixed_quad<P>(r, pb); break;
    case 9: xyzz_add_mixed_pair<P>(r, pb); break;
    case 10: xyzz_shift_quad<P>(r, k); break;
    case 11: case 12: {
        xyzz sum, diff;
        xyzz_addsub_q<P, true>(r, q, sum, diff);
        r = op == 11 ? sum : diff;
        break;
    }
    default: xyzz_double_q<P>(r); break;
    }
    uint32_t differ = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) {
        differ |= r.x.v[j] ^ __shfl_sync(0xffffffffu, r.x.v[j], 0, lanes);
        differ |= r.y.v[j] ^ __shfl_sync(0xffffffffu, r.y.v[j], 0, lanes);
        differ |= r.zz.v[j] ^ __shfl_sync(0xffffffffu, r.zz.v[j], 0, lanes);
        differ |= r.zzz.v[j] ^ __shfl_sync(0xffffffffu, r.zzz.v[j], 0, lanes);
    }
    for (uint32_t o = 1; o < lanes; o <<= 1) differ |= __shfl_xor_sync(0xffffffffu, differ, o, lanes);
    if (i >= n || (threadIdx.x & (lanes - 1))) return;
    st_canonical<P>(out + i, differ ? poison_point<P>() : xyzz_to_affine_dev<P>(r));
}
// throughput microbenchmark: 4 independent dependent-chains per thread
template <class P, bool SQR> __global__ void bench_mul_kernel(fe *io, uint32_t iters) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    fe a = fe_load(io + 4 * i), b = fe_load(io + 4 * i + 1), c = fe_load(io + 4 * i + 2), d = fe_load(io + 4 * i + 3);
    for (uint32_t k = 0; k < iters; k++) {
        if (SQR) { a = fe_sqr<P>(a); b = fe_sqr<P>(b); c = fe_sqr<P>(c); d = fe_sqr<P>(d); }
        else { a = fe_mul<P>(a, b); b = fe_mul<P>(b, c); c = fe_mul<P>(c, d); d = fe_mul<P>(d, a); }
    }
    fe_store(io + 4 * i, a); fe_store(io + 4 * i + 1, b); fe_store(io + 4 * i + 2, c); fe_store(io + 4 * i + 3, d);
}
// single-warp latency microbenchmark of the serial building blocks (tails of the MSM)
template <class P> __global__ void bench_latency_kernel(fe *io, uint32_t iters, int mode) {
    uint32_t i = threadIdx.x;
    fe a = fe_load(io + 4 * i), b = fe_load(io + 4 * i + 1), c = fe_load(io + 4 * i + 2), d = fe_load(io + 4 * i + 3);
    a.v[7] &= 0x3fffffffu; b.v[7] &= 0x3fffffffu; c.v[7] &= 0x3fffffffu; d.v[7] &= 0x3fffffffu;
    if (mode == 0) { for (uint32_t k = 0; k < iters; k++) a = fe_mul<P>(a, b); }
    else if (mode == 1) { for (uint32_t k = 0; k < iters; k++) { a = fe_mul<P>(a, b); c = fe_mul<P>(c, d); } }
    else if (mode == 2) { for (uint32_t k = 0; k < iters; k++) { a = fe_mul<P>(a, b); b = fe_mul<P>(b, c); c = fe_mul<P>(c, d); d = fe_mul<P>(d, a); } }
    else if (mode == 6) { for (uint32_t k = 0; k < iters; k++) { fe_mul2<P>(a, a, b, c, c, d); } }
    else {
        affine g; g.x = fe_neg<P>(fe_one<P>()); g.y = fe_dbl<P>(fe_one<P>());
        xyzz acc = xyzz_double_affine<P>(g), other = acc; xyzz_double<P>(other);
        if (mode == 3) { for (uint32_t k = 0; k < iters; k++) xyzz_double<P>(acc); }
        else if (mode == 4) { for (uint32_t k = 0; k < iters; k++) xyzz_add<P>(acc, other); }
        else { for (uint32_t k = 0; k < iters; k++) xyzz_add_mixed<P>(acc, g); }
        a = acc.x; b = acc.y; c = acc.zz; d = acc.zzz;
    }
    fe_store(io + 4 * i, a); fe_store(io + 4 * i + 1, b); fe_store(io + 4 * i + 2, c); fe_store(io + 4 * i + 3, d);
}
template <class P> __global__ void point_sum_kernel(const jacobian *pts, uint32_t g, int canonical, jacobian *out) {
    if (threadIdx.x || blockIdx.x) return;
    xyzz acc = xyzz_identity();
    for (uint32_t i = 0; i < g; i++) {
        jacobian j;
        j.x = fe_load(&pts[i].x); j.y = fe_load(&pts[i].y); j.z = fe_load(&pts[i].z);
        if (canonical) { j.x = fe_to_mont<P>(j.x); j.y = fe_to_mont<P>(j.y); j.z = fe_to_mont<P>(j.z); }
        xyzz t;
        if (fe_is_zero(j.z)) t = xyzz_identity();
        else { t.x = j.x; t.y = j.y; t.zz = fe_sqr<P>(j.z); t.zzz = fe_mul<P>(t.zz, j.z); }
        xyzz_add<P>(acc, t);
    }
    jacobian r = xyzz_to_jacobian<P>(acc);
    if (canonical) { r.x = fe_from_mont<P>(r.x); r.y = fe_from_mont<P>(r.y); r.z = fe_from_mont<P>(r.z); }
    st_jacobian(out, r);
}

