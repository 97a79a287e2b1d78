// TEST-ONLY host build of the device field/curve headers (PTX carry flag emulated).
// Never loaded by the halo2_b200 package; see tests/kernel_emul/README.md.
#include <cstring>
#include "field.cuh"
#include "curve.cuh"
using namespace h2;

template <class P> static void field_op(int op, const uint8_t *a, const uint8_t *b, uint8_t *out) {
    fe x, y, r;
    memcpy(x.v, a, 32); memcpy(y.v, b, 32);
    x = fe_to_mont<P>(x); y = fe_to_mont<P>(y);
    switch (op) {
    case 0: r = fe_add<P>(x, y); break;
    case 1: r = fe_sub<P>(x, y); break;
    case 2: r = fe_mul<P>(x, y); break;
    case 3: r = fe_inv<P>(x); break;
    case 4: r = fe_sqr<P>(x); break;
    case 5: r = fe_neg<P>(x); break;
    case 6: r = fe_dbl<P>(x); break;
    case 7: r = fe_inv_gcd<P>(x); break;
    default: r = fe_zero();
    }
    r = fe_from_mont<P>(r);
    memcpy(out, r.v, 32);
}
extern "C" int emu_field_op(int field, int op, const uint8_t *a, const uint8_t *b, uint8_t *out) {
    if (field == 0) field_op<FpParams>(op, a, b, out); else field_op<FqParams>(op, a, b, out);
    return 0;
}

// points cross as canonical affine x||y (identity = zeros); op: 0 = xyzz(a)+affine(b) mixed,
// 1 = full add, 2 = double(a), 7 = acc chain: ((a + b) + b) + a via mixed adds,
// 8 = scalar mul by 32-byte LE scalar in b[0..32) via the device double-and-add helper.
// 3 .. 6 = the serial ops of h2_test_curve_op on the same rescaled operands (test_lambda of element i): 3 xyzz_add, 4 xyzz_add_mixed,
// 5 xyzz_double, 6 xyzz_shift by the low 32 bits of b.x.
template <class P> static void load_aff(affine &r, const uint8_t *b) {
    memcpy(r.x.v, b, 32); memcpy(r.y.v, b + 32, 32);
    if (!(fe_is_zero(r.x) && fe_is_zero(r.y))) { r.x = fe_to_mont<P>(r.x); r.y = fe_to_mont<P>(r.y); }
}
template <class P> static void store_xyzz(const xyzz &p, uint8_t *out) {
    jacobian j = xyzz_to_jacobian<P>(p);
    affine a = jacobian_to_affine<P>(j);
    fe x = fe_from_mont<P>(a.x), y = fe_from_mont<P>(a.y);
    memcpy(out, x.v, 32); memcpy(out + 32, y.v, 32);
}
template <class P> static void curve_op(int op, const uint8_t *a, const uint8_t *b, uint64_t i, uint8_t *out) {
    affine pa, pb; load_aff<P>(pa, a);
    xyzz r = xyzz_identity();
    if (op == 8) {
        uint32_t k[8]; memcpy(k, b, 32);
        r = xyzz_scalar_mul<P>(pa, k);
    } else if (op == 6) {
        uint32_t k; memcpy(&k, b, 4);
        r = xyzz_rescale<P>(xyzz_from_affine<P>(pa), test_lambda<P>(i, 0));
        xyzz_shift<P>(r, k);
    } else {
        load_aff<P>(pb, b);
        xyzz xa = xyzz_from_affine<P>(pa), xb = xyzz_from_affine<P>(pb);
        if (op >= 3 && op <= 5) { xa = xyzz_rescale<P>(xa, test_lambda<P>(i, 0)); xb = xyzz_rescale<P>(xb, test_lambda<P>(i, 1)); }
        if (op == 0 || op == 4) { r = xa; xyzz_add_mixed<P>(r, pb); }
        else if (op == 1 || op == 3) { r = xa; xyzz_add<P>(r, xb); }
        else if (op == 2 || op == 5) { r = xa; xyzz_double<P>(r); }
        else if (op == 7) { r = xa; xyzz_add_mixed<P>(r, pb); xyzz_add_mixed<P>(r, pb); xyzz_add_mixed<P>(r, pa); xyzz t = r; xyzz_add<P>(r, t); }
    }
    store_xyzz<P>(r, out);
}
extern "C" int emu_curve_op(int curve, int op, const uint8_t *a, const uint8_t *b, uint64_t i, uint8_t *out) {
    if (curve == 0) curve_op<FpParams>(op, a, b, i, out); else curve_op<FqParams>(op, a, b, i, out);
    return 0;
}

#include "glv.cuh"
// GLV split of a canonical scalar: out = |k1| (32 B) || |k2| (32 B) || neg1 || neg2
extern "C" int emu_glv(int curve, const uint8_t *k, uint8_t *out) {
    uint32_t kk[8], k1[8], k2[8], n1, n2;
    memcpy(kk, k, 32);
    if (curve == 0) glv_decompose<FpParams>(kk, k1, n1, k2, n2); else glv_decompose<FqParams>(kk, k1, n1, k2, n2);
    memcpy(out, k1, 32); memcpy(out + 32, k2, 32); out[64] = (uint8_t)n1; out[65] = (uint8_t)n2;
    return 0;
}
// phi(P) = (zeta x, y) on canonical affine bytes
extern "C" int emu_phi(int curve, const uint8_t *xy, uint8_t *out) {
    fe x; memcpy(x.v, xy, 32);
    if (curve == 0) x = fe_from_mont<FpParams>(fe_mul<FpParams>(fe_to_mont<FpParams>(x), glv_zeta<FpParams>()));
    else x = fe_from_mont<FqParams>(fe_mul<FqParams>(fe_to_mont<FqParams>(x), glv_zeta<FqParams>()));
    memcpy(out, x.v, 32); memcpy(out + 32, xy + 32, 32);
    return 0;
}
