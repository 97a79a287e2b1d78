// Device curve library for Pallas / Vesta, y^2 = x^3 + 5 (K1 in SURVEY.md section 2.1).
//
// Replaces the pasta_curves Ep/Eq group law that the reference's buckets use
// (halo2_proofs/src/arithmetic.rs:37-57 Bucket::add_assign/add, :86-91 running sums,
// :163 window doubling, :166 window sum).  The template parameter is the COORDINATE field
// (FpParams for Pallas, FqParams for Vesta).
//
// Accumulators use extended Jacobian "XYZZ" coordinates (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2):
// mixed add 8M+2S, full add 12M+2S, double 6M+3S, no inversion anywhere on the hot path.
// Identity: affine (0,0) (book/src/background/curves.md:226-230); XYZZ with ZZ == 0.
// Every add handles P+P, P+(-P), identity operands (cf. the reference's msm_arithmetic test,
// poly/commitment/msm.rs:179-219).
#pragma once
#include "field.cuh"

namespace h2 {

struct affine { fe x, y; };              // 64 B, Montgomery coordinates; (0,0) = identity
struct xyzz { fe x, y, zz, zzz; };       // 128 B
struct jacobian { fe x, y, z; };         // 96 B, the layout of pasta's Ep/Eq (x, y, z)

// Out-of-line multiply / square for the group law.  Inlined, one mixed add is ~45 KB of straight-line SASS (a full add
// ~60 KB); with ~20 resident warps at unrelated program counters the instruction caches thrash.  Called, a kernel's group law is a few KB plus the two callees.  Arguments and result travel in
// registers.  cm / cs are what the formulas below use; the host (emulation) build inlines.
#ifdef __CUDA_ARCH__
template <class P> __device__ __noinline__ fe fe_mul_call(fe a, fe b) { return fe_mul<P>(a, b); }
template <class P> __device__ __noinline__ fe fe_sqr_call(fe a) { return fe_sqr<P>(a); }
#else
template <class P> inline fe fe_mul_call(const fe &a, const fe &b) { return fe_mul<P>(a, b); }
template <class P> inline fe fe_sqr_call(const fe &a) { return fe_sqr<P>(a); }
#endif
#define cm fe_mul_call
#define cs fe_sqr_call

H2_HD bool affine_is_identity(const affine &p) {
    uint32_t t = 0;
    for (int i = 0; i < 8; i++) t |= p.x.v[i] | p.y.v[i];
    return t == 0;
}
H2_HD xyzz xyzz_identity() {
    xyzz r; r.x = fe_zero(); r.y = fe_zero(); r.zz = fe_zero(); r.zzz = fe_zero();
    return r;
}
H2_HD bool xyzz_is_identity(const xyzz &p) { return fe_is_zero(p.zz); }

template <class P> H2_HD xyzz xyzz_from_affine(const affine &p) {
    xyzz r;
    if (affine_is_identity(p)) return xyzz_identity();
    r.x = p.x; r.y = p.y; r.zz = fe_one<P>(); r.zzz = fe_one<P>();
    return r;
}
// The same point in another representation: (l^2 X, l^3 Y, l^2 ZZ, l^3 ZZZ) for l != 0; the identity stays (0, 0, 0, 0).
// Only the group-law self-tests use it (h2_test_curve_op, tests/kernel_emul), to give every form operands with ZZ != 1.
template <class P> H2_HD xyzz xyzz_rescale(const xyzz &p, const fe &l) {
    if (xyzz_is_identity(p)) return xyzz_identity();
    const fe l2 = fe_sqr<P>(l), l3 = fe_mul<P>(l2, l);
    xyzz r;
    r.x = fe_mul<P>(p.x, l2); r.y = fe_mul<P>(p.y, l3); r.zz = fe_mul<P>(p.zz, l2); r.zzz = fe_mul<P>(p.zzz, l3);
    return r;
}
H2_HD uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}
// The rescaling factor of operand `which` of self-test element i: 1 for i % 4 == 0 (the ZZ = 1 case stays covered), otherwise
// a non-zero field element below 2^254 mixed from (i, which) -- the device kernel and its host emulation draw the same one.
template <class P> H2_HD fe test_lambda(uint64_t i, uint32_t which) {
    if (i % 4 == 0) return fe_one<P>();
    fe l;
    uint64_t s = splitmix64(i * 2 + which);
    for (int j = 0; j < 8; j += 2) {
        s = splitmix64(s);
        l.v[j] = (uint32_t)s; l.v[j + 1] = (uint32_t)(s >> 32);
    }
    l.v[7] &= 0x3fffffffu;
    if (fe_is_zero(l)) l = fe_one<P>();
    return l;
}
template <class P> H2_HD void xyzz_neg(xyzz &p) { p.y = fe_neg<P>(p.y); }
template <class P> H2_HD affine affine_neg(const affine &p) {
    affine r; r.x = p.x; r.y = fe_neg<P>(p.y);   // -(0,0) = (0,0): fe_neg(0) = 0
    return r;
}

// 2 * (affine p) -> XYZZ   (mdbl-2008-s-1, a = 0)
template <class P> H2_HD xyzz xyzz_double_affine(const affine &p) {
    xyzz r;
    fe u = fe_dbl<P>(p.y);
    fe v = cs<P>(u);
    fe w = cm<P>(u, v);
    fe s = cm<P>(p.x, v);
    fe m = cs<P>(p.x);
    m = fe_add<P>(fe_dbl<P>(m), m);
    r.x = fe_sub<P>(fe_sub<P>(cs<P>(m), s), s);
    r.y = fe_sub<P>(cm<P>(m, fe_sub<P>(s, r.x)), cm<P>(w, p.y));
    r.zz = v; r.zzz = w;
    return r;
}

// acc = 2 * acc   (dbl-2008-s-1, a = 0)
template <class P> H2_HD void xyzz_double(xyzz &a) {
    if (xyzz_is_identity(a)) return;
    fe u = fe_dbl<P>(a.y);
    fe v = cs<P>(u);
    fe w = cm<P>(u, v);
    fe s = cm<P>(a.x, v);
    fe m = cs<P>(a.x);
    m = fe_add<P>(fe_dbl<P>(m), m);
    fe x3 = fe_sub<P>(fe_sub<P>(cs<P>(m), s), s);
    fe y3 = fe_sub<P>(cm<P>(m, fe_sub<P>(s, x3)), cm<P>(w, a.y));
    a.x = x3; a.y = y3;
    a.zz = cm<P>(v, a.zz);
    a.zzz = cm<P>(w, a.zzz);
}

// acc += affine p   (madd-2008-s); the hot operation of the bucket accumulation
template <class P> H2_HD void xyzz_add_mixed(xyzz &a, const affine &p) {
    if (affine_is_identity(p)) return;
    if (xyzz_is_identity(a)) { a = xyzz_from_affine<P>(p); return; }
    fe u2 = cm<P>(p.x, a.zz);
    fe s2 = cm<P>(p.y, a.zzz);
    fe pp = fe_sub<P>(u2, a.x);
    fe r = fe_sub<P>(s2, a.y);
    if (fe_is_zero(pp)) {
        if (fe_is_zero(r)) a = xyzz_double_affine<P>(p);   // same point
        else a = xyzz_identity();                          // opposite points
        return;
    }
    fe pp2 = cs<P>(pp);
    fe ppp = cm<P>(pp, pp2);
    fe q = cm<P>(a.x, pp2);
    fe x3 = fe_sub<P>(fe_sub<P>(fe_sub<P>(cs<P>(r), ppp), q), q);
    fe y3 = fe_sub<P>(cm<P>(r, fe_sub<P>(q, x3)), cm<P>(a.y, ppp));
    a.x = x3; a.y = y3;
    a.zz = cm<P>(a.zz, pp2);
    a.zzz = cm<P>(a.zzz, ppp);
}

// acc += b   (add-2008-s)
template <class P> H2_HD void xyzz_add(xyzz &a, const xyzz &b) {
    if (xyzz_is_identity(b)) return;
    if (xyzz_is_identity(a)) { a = b; return; }
    fe u1 = cm<P>(a.x, b.zz);
    fe u2 = cm<P>(b.x, a.zz);
    fe s1 = cm<P>(a.y, b.zzz);
    fe s2 = cm<P>(b.y, a.zzz);
    fe pp = fe_sub<P>(u2, u1);
    fe r = fe_sub<P>(s2, s1);
    if (fe_is_zero(pp)) {
        if (fe_is_zero(r)) xyzz_double<P>(a);
        else a = xyzz_identity();
        return;
    }
    fe pp2 = cs<P>(pp);
    fe ppp = cm<P>(pp, pp2);
    fe q = cm<P>(u1, pp2);
    fe x3 = fe_sub<P>(fe_sub<P>(fe_sub<P>(cs<P>(r), ppp), q), q);
    fe y3 = fe_sub<P>(cm<P>(r, fe_sub<P>(q, x3)), cm<P>(s1, ppp));
    a.x = x3; a.y = y3;
    a.zz = cm<P>(cm<P>(a.zz, b.zz), pp2);
    a.zzz = cm<P>(cm<P>(a.zzz, b.zzz), ppp);
}

// XYZZ -> Jacobian without inversion: (X*ZZ, Y*ZZZ, ZZ) since (ZZ)^2 * x = X*ZZ and
// (ZZ)^3 * y = ZZZ^2 * y = Y*ZZZ.  Identity maps to z = 0 (pasta: (0, 1, 0)-like).
template <class P> H2_HD jacobian xyzz_to_jacobian(const xyzz &p) {
    jacobian j;
    if (xyzz_is_identity(p)) { j.x = fe_zero(); j.y = fe_one<P>(); j.z = fe_zero(); return j; }
    j.x = cm<P>(p.x, p.zz);
    j.y = cm<P>(p.y, p.zzz);
    j.z = p.zz;
    return j;
}
template <class P> H2_HD affine jacobian_to_affine(const jacobian &j) {
    affine r;
    if (fe_is_zero(j.z)) { r.x = fe_zero(); r.y = fe_zero(); return r; }
    fe zi = fe_inv_gcd<P>(j.z);
    fe zi2 = cs<P>(zi);
    r.x = cm<P>(j.x, zi2);
    r.y = cm<P>(j.y, cm<P>(zi2, zi));
    return r;
}

// acc = 2^k * acc through Jacobian coordinates: the a = 0 doubling dbl-2009-l costs 2M + 5S
// (XYZZ doubling: 6M + 3S), which pays off on the long shift chains of the window combine.  That chain is run by lone
// warps (pure latency), so its multiplies stay inlined: a call adds latency to every multiply when nothing else hides it.
template <class P> H2_HD void xyzz_shift(xyzz &a, uint32_t k) {
    if (k == 0 || xyzz_is_identity(a)) return;
    if (k < 4) { for (uint32_t d = 0; d < k; d++) xyzz_double<P>(a); return; }
    fe X = fe_mul<P>(a.x, a.zz), Y = fe_mul<P>(a.y, a.zzz), Z = a.zz;   // (X ZZ, Y ZZZ, ZZ)
    for (uint32_t d = 0; d < k; d++) {
        fe A = fe_sqr<P>(X), B = fe_sqr<P>(Y), C = fe_sqr<P>(B);
        fe t = fe_add<P>(X, B);
        fe D = fe_sub<P>(fe_sub<P>(fe_sqr<P>(t), A), C);
        D = fe_dbl<P>(D);
        fe E = fe_add<P>(fe_dbl<P>(A), A);
        fe F = fe_sqr<P>(E);
        fe Z3 = fe_dbl<P>(fe_mul<P>(Y, Z));
        X = fe_sub<P>(fe_sub<P>(F, D), D);
        fe C8 = fe_dbl<P>(fe_dbl<P>(fe_dbl<P>(C)));
        Y = fe_sub<P>(fe_mul<P>(E, fe_sub<P>(D, X)), C8);
        Z = Z3;
    }
    // Jacobian (X, Y, Z) -> XYZZ (X, Y, Z^2, Z^3); Y == 0 cannot occur on a prime-order curve
    a.x = X; a.y = Y;
    a.zz = fe_sqr<P>(Z);
    a.zzz = fe_mul<P>(a.zz, Z);
}

#ifdef __CUDACC__
// xyzz_shift for a QUAD: four consecutive lanes hold the same point and call this together.  A Jacobian doubling is
// 7 multiplies but only 3 deep -- (X^2, Y^2, Y Z) -> (B^2, (X + B)^2, E^2) -> E (D - X3) -- so lanes 0..2 each take one
// product of a level and the quad exchanges the results by shuffle; the last product is computed redundantly.  The
// serial doubling chain of the window combine (c (W - 1) + ~15 doublings for the top window, nothing else to overlap
// it with) shortens from 7 to 3 multiply latencies per step.
H2_D fe quad_bcast(const fe &v, uint32_t src, uint32_t mask) {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_sync(mask, v.v[i], src, 4);
    return r;
}
H2_D fe fe_select(bool c, const fe &a, const fe &b) {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = c ? a.v[i] : b.v[i];
    return r;
}
// acc += b for a QUAD (four consecutive lanes holding the same a and b).  The 14 multiplies of add-2008-s are 4 deep:
//   (u1, u2, s1, s2) -> (pp^2, r^2, zz zz', zzz zzz') -> (pp^3, q, zz3) -> (r (q - x3), s1 pp^3, zzz3)
// one product per lane and level, results exchanged by shuffle.  Same lane-multiplies as the serial form, 4 multiply
// latencies instead of 14 -- for the bucket-reduce / tree kernels, whose serial chains of additions are latency-bound.
template <class P> H2_D void xyzz_add_quad(xyzz &a, const xyzz &b) {
    if (xyzz_is_identity(b)) return;                     // all tests are uniform within the quad
    if (xyzz_is_identity(a)) { a = b; return; }
    const uint32_t lane = threadIdx.x & 31u, sub = lane & 3u, mask = 0xFu << (lane & ~3u);
    const bool s0 = sub == 0, s1_ = sub == 1, s2_ = sub == 2;
    // level 1: u1 = a.x b.zz | u2 = b.x a.zz | s1 = a.y b.zzz | s2 = b.y a.zzz
    fe r_ = fe_mul<P>(fe_select(s0, a.x, fe_select(s1_, b.x, fe_select(s2_, a.y, b.y))),
                      fe_select(s0, b.zz, fe_select(s1_, a.zz, fe_select(s2_, b.zzz, a.zzz))));
    fe u1 = quad_bcast(r_, 0, mask), u2 = quad_bcast(r_, 1, mask), s1 = quad_bcast(r_, 2, mask), s2 = quad_bcast(r_, 3, mask);
    fe pp = fe_sub<P>(u2, u1);
    fe r = fe_sub<P>(s2, s1);
    if (fe_is_zero(pp)) {
        if (fe_is_zero(r)) xyzz_double<P>(a);
        else a = xyzz_identity();
        return;
    }
    // level 2: pp^2 | r^2 | a.zz b.zz | a.zzz b.zzz
    r_ = fe_mul<P>(fe_select(s0, pp, fe_select(s1_, r, fe_select(s2_, a.zz, a.zzz))),
                   fe_select(s0, pp, fe_select(s1_, r, fe_select(s2_, b.zz, b.zzz))));
    fe pp2 = quad_bcast(r_, 0, mask), rr = quad_bcast(r_, 1, mask), zz12 = quad_bcast(r_, 2, mask), zzz12 = quad_bcast(r_, 3, mask);
    // level 3: pp^3 | q = u1 pp^2 | zz3 = zz12 pp^2
    r_ = fe_mul<P>(fe_select(s0, pp, fe_select(s1_, u1, zz12)), pp2);
    fe ppp = quad_bcast(r_, 0, mask), q = quad_bcast(r_, 1, mask), zz3 = quad_bcast(r_, 2, mask);
    fe x3 = fe_sub<P>(fe_sub<P>(fe_sub<P>(rr, ppp), q), q);
    // level 4: r (q - x3) | s1 pp^3 | zzz3 = zzz12 pp^3
    r_ = fe_mul<P>(fe_select(s0, r, fe_select(s1_, s1, zzz12)), fe_select(s0, fe_sub<P>(q, x3), ppp));
    fe t1 = quad_bcast(r_, 0, mask), t2 = quad_bcast(r_, 1, mask), zzz3 = quad_bcast(r_, 2, mask);
    a.x = x3; a.y = fe_sub<P>(t1, t2);
    a.zz = zz3; a.zzz = zzz3;
}
// acc += affine p for a QUAD (madd-2008-s, 8M + 2S, 4 levels deep):
//   (u2, s2) -> (pp^2, r^2) -> (pp^3, q, zz3) -> (r (q - x3), y1 pp^3, zzz3)
// for SMALL accumulations (k <= 16 commits, IPA rounds), where the kernel's duration is the longest bucket's serial chain.
template <class P> H2_D void xyzz_add_mixed_quad(xyzz &a, const affine &p) {
    if (affine_is_identity(p)) return;                   // all tests are uniform within the quad
    if (xyzz_is_identity(a)) { a = xyzz_from_affine<P>(p); return; }
    const uint32_t lane = threadIdx.x & 31u, sub = lane & 3u, mask = 0xFu << (lane & ~3u);
    const bool s0 = sub == 0, s1_ = sub == 1;
    // level 1: u2 = p.x a.zz | s2 = p.y a.zzz
    fe r_ = fe_mul<P>(fe_select(s0, p.x, p.y), fe_select(s0, a.zz, a.zzz));
    fe u2 = quad_bcast(r_, 0, mask), s2 = quad_bcast(r_, 1, mask);
    fe pp = fe_sub<P>(u2, a.x);
    fe r = fe_sub<P>(s2, a.y);
    if (fe_is_zero(pp)) {
        if (fe_is_zero(r)) a = xyzz_double_affine<P>(p);   // same point
        else a = xyzz_identity();                          // opposite points
        return;
    }
    // level 2: pp^2 | r^2
    r_ = fe_sqr<P>(fe_select(s0, pp, r));
    fe pp2 = quad_bcast(r_, 0, mask), rr = quad_bcast(r_, 1, mask);
    // level 3: pp^3 | q = a.x pp^2 | zz3 = a.zz pp^2
    r_ = fe_mul<P>(fe_select(s0, pp, fe_select(s1_, a.x, a.zz)), pp2);
    fe ppp = quad_bcast(r_, 0, mask), q = quad_bcast(r_, 1, mask), zz3 = quad_bcast(r_, 2, mask);
    fe x3 = fe_sub<P>(fe_sub<P>(fe_sub<P>(rr, ppp), q), q);
    // level 4: r (q - x3) | a.y pp^3 | zzz3 = a.zzz pp^3
    r_ = fe_mul<P>(fe_select(s0, r, fe_select(s1_, a.y, a.zzz)), fe_select(s0, fe_sub<P>(q, x3), ppp));
    fe t1 = quad_bcast(r_, 0, mask), t2 = quad_bcast(r_, 1, mask), zzz3 = quad_bcast(r_, 2, mask);
    a.x = x3; a.y = fe_sub<P>(t1, t2);
    a.zz = zz3; a.zzz = zzz3;
}
// acc += affine p for a PAIR of lanes (lanes 2 i and 2 i + 1 hold the same a and p).  The 10 products of madd-2008-s split
// into five levels of two -- (u2, s2) -> (pp^2, r^2) -> (pp^3, q) -> (zz3, y1 pp^3) -> (r (q - x3), zzz3) -- so a pair spends
// exactly 10 lane-multiplies per addition (a quad: 16 slots for 10 products) at 5 multiply latencies (a quad: 4, one lane:
// 10).  For the small accumulations whose kernel is bound by lane-multiplies AND by its longest chain (k <= 16 commits, IPA rounds).
template <class P> H2_D void xyzz_add_mixed_pair(xyzz &a, const affine &p) {
    if (affine_is_identity(p)) return;                   // all tests are uniform within the pair
    if (xyzz_is_identity(a)) { a = xyzz_from_affine<P>(p); return; }
    const uint32_t lane = threadIdx.x & 31u, mask = 0x3u << (lane & ~1u);
    const bool s0 = (lane & 1u) == 0;
    auto swap = [&](const fe &mine, fe &first, fe &second) {   // first = lane 0's product, second = lane 1's
        fe other;
#pragma unroll
        for (int i = 0; i < 8; i++) other.v[i] = __shfl_xor_sync(mask, mine.v[i], 1);
        first = fe_select(s0, mine, other); second = fe_select(s0, other, mine);
    };
    fe u2, s2, pp2, rr, ppp, q, zz3, t2, t1, zzz3;
    swap(fe_mul<P>(fe_select(s0, p.x, p.y), fe_select(s0, a.zz, a.zzz)), u2, s2);
    const fe pp = fe_sub<P>(u2, a.x), r = fe_sub<P>(s2, a.y);
    if (fe_is_zero(pp)) {
        if (fe_is_zero(r)) a = xyzz_double_affine<P>(p);   // same point
        else a = xyzz_identity();                          // opposite points
        return;
    }
    swap(fe_sqr<P>(fe_select(s0, pp, r)), pp2, rr);
    swap(fe_mul<P>(fe_select(s0, pp, a.x), pp2), ppp, q);
    const fe x3 = fe_sub<P>(fe_sub<P>(fe_sub<P>(rr, ppp), q), q);
    swap(fe_mul<P>(fe_select(s0, a.zz, a.y), fe_select(s0, pp2, ppp)), zz3, t2);
    swap(fe_mul<P>(fe_select(s0, r, a.zzz), fe_select(s0, fe_sub<P>(q, x3), ppp)), t1, zzz3);
    a.x = x3; a.y = fe_sub<P>(t1, t2);
    a.zz = zz3; a.zzz = zzz3;
}
template <class P> H2_D void xyzz_shift_quad(xyzz &a, uint32_t k) {
    if (k == 0 || xyzz_is_identity(a)) return;          // uniform within the quad
    const uint32_t lane = threadIdx.x & 31u, sub = lane & 3u, mask = 0xFu << (lane & ~3u);
    fe X = fe_mul<P>(a.x, a.zz), Y = fe_mul<P>(a.y, a.zzz), Z = a.zz;   // Jacobian (X ZZ, Y ZZZ, ZZ)
    for (uint32_t d = 0; d < k; d++) {
        fe r = fe_mul<P>(fe_select(sub == 0, X, Y), fe_select(sub == 0, X, fe_select(sub == 1, Y, Z)));
        fe A = quad_bcast(r, 0, mask), B = quad_bcast(r, 1, mask), YZ = quad_bcast(r, 2, mask);
        fe E = fe_add<P>(fe_dbl<P>(A), A);
        fe t = fe_add<P>(X, B);
        r = fe_sqr<P>(fe_select(sub == 0, B, fe_select(sub == 1, t, E)));
        fe C = quad_bcast(r, 0, mask), T2 = quad_bcast(r, 1, mask), F = quad_bcast(r, 2, mask);
        fe D = fe_dbl<P>(fe_sub<P>(fe_sub<P>(T2, A), C));
        X = fe_sub<P>(fe_sub<P>(F, D), D);
        fe C8 = fe_dbl<P>(fe_dbl<P>(fe_dbl<P>(C)));
        Y = fe_sub<P>(fe_mul<P>(E, fe_sub<P>(D, X)), C8);
        Z = fe_dbl<P>(YZ);
    }
    a.x = X; a.y = Y;
    a.zz = fe_sqr<P>(Z);
    a.zzz = fe_mul<P>(a.zz, Z);
}
#endif

// k * p by left-to-right double-and-add; k = 8 x u32 little-endian (canonical integer).
// Used by the synthetic-input generator and the tests, not by the MSM hot path.
template <class P> H2_HD xyzz xyzz_scalar_mul(const affine &p, const uint32_t (&k)[8]) {
    xyzz acc = xyzz_identity();
    for (int i = 7; i >= 0; i--) {
        for (int b = 31; b >= 0; b--) {
            xyzz_double<P>(acc);
            if ((k[i] >> b) & 1u) xyzz_add_mixed<P>(acc, p);
        }
    }
    return acc;
}

#undef cm
#undef cs

}  // namespace h2
