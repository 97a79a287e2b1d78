//! Safe wrappers over include/halo2_b200.h for halo2_proofs.
//!
//! halo2_proofs forbids `unsafe` (`src/lib.rs:9`), so the FFI lives in this separate crate and
//! halo2_proofs::arithmetic dispatches into it on the concrete Pasta types (see INTEGRATION.md).
//! Element encoding: the portable canonical path (`to_repr` / `coordinates`) is always correct;
//! the zero-copy Montgomery path is enabled only after `self_test()` confirms that pasta_curves'
//! in-memory layout is 4 x u64 little-endian Montgomery limbs with R = 2^256.
#![allow(clippy::missing_safety_doc)]
use std::ffi::CStr;
use std::os::raw::{c_char, c_int, c_void};

use ff::PrimeField;
use group::Curve;
use pasta_curves::arithmetic::{CurveAffine, CurveExt};
use pasta_curves::{pallas, vesta};

pub const CURVE_PALLAS: c_int = 0;
pub const CURVE_VESTA: c_int = 1;
pub const FIELD_FP: c_int = 0;
pub const FIELD_FQ: c_int = 1;
pub const REPR_CANONICAL: c_int = 0;
pub const REPR_MONTGOMERY: c_int = 1;

extern "C" {
    pub fn h2_init(device: c_int) -> c_int;
    pub fn h2_last_error() -> *const c_char;
    pub fn h2_msm(curve: c_int, scalars: *const c_void, bases_xy: *const c_void, n: usize, repr: c_int,
                  out_xyz: *mut c_void) -> c_int;
    pub fn h2_bases_register(curve: c_int, bases_xy: *const c_void, n: usize, repr: c_int, handle: *mut u64) -> c_int;
    pub fn h2_bases_register_ex(curve: c_int, bases_xy: *const c_void, n: usize, repr: c_int, window_bits: u32, flags: u32,
                                handle: *mut u64) -> c_int;
    pub fn h2_bases_release(handle: u64) -> c_int;
    pub fn h2_msm_registered_batch(handle: u64, scalars: *const c_void, n: usize, extra_scalars: *const c_void, batch: usize,
                                   repr: c_int, out_xyz: *mut c_void) -> c_int;
    pub fn h2_poly_alloc(field: c_int, len: usize, poly: *mut u64) -> c_int;
    pub fn h2_poly_free(poly: u64) -> c_int;
    pub fn h2_poly_upload(poly: u64, src: *const c_void, len: usize, repr: c_int) -> c_int;
    pub fn h2_poly_download(poly: u64, dst: *mut c_void, len: usize, repr: c_int) -> c_int;
    pub fn h2_poly_lagrange_to_coeff(dst: u64, src: u64, k: u32, omega_inv: *const c_void, divisor: *const c_void, repr: c_int) -> c_int;
    pub fn h2_poly_coeff_to_extended(dst: u64, src: u64, k: u32, ext_k: u32, zeta: *const c_void, ext_omega: *const c_void,
                                     repr: c_int) -> c_int;
    pub fn h2_poly_extended_to_coeff(dst: u64, src: u64, ext_k: u32, ext_omega_inv: *const c_void, ext_divisor: *const c_void,
                                     zeta: *const c_void, out_len: usize, repr: c_int) -> c_int;
    pub fn h2_msm_registered_polys(bases_handle: u64, polys: *const u64, batch: usize, n: usize, extra_scalars: *const c_void,
                                   repr: c_int, out_xyz: *mut c_void) -> c_int;
    pub fn h2_ipa_begin(bases_handle: u64, k: u32, p_prime: *const c_void, x3: *const c_void, repr: c_int, session: *mut u64) -> c_int;
    pub fn h2_ipa_round(session: u64, z: *const c_void, l_rand: *const c_void, r_rand: *const c_void, repr: c_int,
                        out_lr_xyz: *mut c_void) -> c_int;
    pub fn h2_ipa_fold(session: u64, u: *const c_void, u_inv: *const c_void, repr: c_int) -> c_int;
    pub fn h2_ipa_finish(session: u64, repr: c_int, out_c_b: *mut c_void) -> c_int;
    pub fn h2_msm_registered(handle: u64, scalars: *const c_void, n: usize, extra_scalar: *const c_void,
                             repr: c_int, out_xyz: *mut c_void) -> c_int;
    pub fn h2_ntt(field: c_int, a: *mut c_void, omega: *const c_void, log_n: u32, repr: c_int) -> c_int;
    pub fn h2_intt_scaled(field: c_int, a: *mut c_void, omega_inv: *const c_void, divisor: *const c_void,
                          log_n: u32, repr: c_int) -> c_int;
    pub fn h2_coeff_to_extended(field: c_int, a: *const c_void, k: u32, ext_k: u32, zeta: *const c_void,
                                ext_omega: *const c_void, out: *mut c_void, repr: c_int) -> c_int;
    pub fn h2_extended_to_coeff(field: c_int, a: *const c_void, ext_k: u32, ext_omega_inv: *const c_void,
                                ext_divisor: *const c_void, zeta: *const c_void, out_len: usize,
                                out: *mut c_void, repr: c_int) -> c_int;
    pub fn h2_ec_fft(curve: c_int, points_xyz: *mut c_void, omega: *const c_void, log_n: u32, scale: *const c_void, repr: c_int) -> c_int;
    pub fn h2_batch_normalize(curve: c_int, points_xyz: *const c_void, n: usize, repr: c_int, out_xy: *mut c_void) -> c_int;
    pub fn h2_poly_eval_ast(out: u64, polys: *const u64, n_polys: usize, log_n: u32, code: *const u32, n_code: usize, consts: *const c_void,
                            n_consts: usize, omega: *const c_void, lin_base: *const c_void, repr: c_int) -> c_int;
    pub fn h2_poly_batch_invert(poly: u64, n: usize) -> c_int;
    pub fn h2_poly_running_product(dst: u64, src: u64, n: usize, init: *const c_void, repr: c_int) -> c_int;
    // the verifier's MSM with resident g_scalars: compute_s (poly/commitment/verifier.rs:156-171) and MSM::scale / add_msm (msm.rs:37-139)
    pub fn h2_poly_compute_s(dst: u64, u: *const c_void, k: u32, init: *const c_void, accumulate: c_int, repr: c_int) -> c_int;
    pub fn h2_poly_scale_add(dst: u64, a: *const c_void, src: u64, b: *const c_void, n: usize, repr: c_int) -> c_int;
    // keygen: the permutation polynomials from the copy-constraint mapping (plonk/permutation/keygen.rs:102-211)
    pub fn h2_poly_permutation_sigma(dst: *const u64, cols: usize, k: u32, mapping: *const u32, omega: *const c_void, delta: *const c_void,
                                     repr: c_int) -> c_int;
    // the same polynomials from the copy constraints: Assembly::copy's cycles computed on the device (plonk/permutation/keygen.rs:45-100)
    pub fn h2_poly_permutation_sigma_copies(dst: *const u64, cols: usize, k: u32, copies: *const u32, m: usize, omega: *const c_void,
                                            delta: *const c_void, repr: c_int) -> c_int;
    pub fn h2_poly_divide_by_vanishing(poly: u64, ext_k: u32, t_evals: *const c_void, t_len: u32, repr: c_int) -> c_int;
    // h(X) divided, transformed back and split into `count` pieces of 2^k coefficients in one call (plonk/vanishing/prover.rs:84-100)
    pub fn h2_poly_vanishing_quotient(pieces: *const u64, count: usize, src: u64, k: u32, ext_k: u32, ext_omega_inv: *const c_void,
                                      ext_divisor: *const c_void, zeta: *const c_void, t_evals: *const c_void, t_len: u32, repr: c_int) -> c_int;
    pub fn h2_poly_eval(polys: *const u64, batch: usize, n: usize, points: *const c_void, repr: c_int, out: *mut c_void) -> c_int;
    pub fn h2_poly_inner_product(a: *const u64, b: *const u64, batch: usize, n: usize, repr: c_int, out: *mut c_void) -> c_int;
    pub fn h2_poly_kate_division(dst: *const u64, src: *const u64, batch: usize, n: usize, points: *const c_void, repr: c_int) -> c_int;
    pub fn h2_points_compress(curve: c_int, points_xy: *const c_void, n: usize, repr: c_int, out_bytes: *mut c_void) -> c_int;
    pub fn h2_points_decompress(curve: c_int, bytes: *const c_void, n: usize, repr: c_int, out_xy: *mut c_void) -> c_int;
    pub fn h2_params_lagrange(curve: c_int, g_xy: *const c_void, k: u32, omega_inv: *const c_void, minv: *const c_void, repr: c_int,
                              out_g_lagrange_xy: *mut c_void) -> c_int;
    // round 2
    pub fn h2_hash_to_curve(curve: c_int, domain_prefix: *const c_char, messages: *const c_void, msg_len: usize, n: usize, repr: c_int,
                            out_xy: *mut c_void) -> c_int;
    pub fn h2_params_new(curve: c_int, k: u32, repr: c_int, out_g_xy: *mut c_void, out_g_lagrange_xy: *mut c_void, out_w_xy: *mut c_void,
                         out_u_xy: *mut c_void) -> c_int;
    pub fn h2_msm_registered_batch_affine(handle: u64, scalars: *const c_void, n: usize, extra_scalars: *const c_void, batch: usize,
                                          repr: c_int, out_xy: *mut c_void) -> c_int;
    pub fn h2_msm_registered_polys_affine(bases_handle: u64, polys: *const u64, batch: usize, n: usize, extra_scalars: *const c_void,
                                          repr: c_int, out_xy: *mut c_void) -> c_int;
    pub fn h2_ipa_begin_poly(bases_handle: u64, k: u32, p_prime_poly: u64, x3: *const c_void, repr: c_int, session: *mut u64) -> c_int;
    pub fn h2_ipa_round_affine(session: u64, z: *const c_void, l_rand: *const c_void, r_rand: *const c_void, repr: c_int,
                               out_lr_xy: *mut c_void) -> c_int;
    pub fn h2_poly_add_at(poly: u64, index: usize, delta: *const c_void, repr: c_int) -> c_int;
    pub fn h2_poly_copy(dst: u64, dst_off: usize, src: u64, src_off: usize, len: usize) -> c_int;
    pub fn h2_poly_lookup_permute(input: u64, table: u64, usable_rows: usize, out_input: u64, out_table: u64) -> c_int;
    pub fn h2_multi_init(ngpu: c_int) -> c_int;
    pub fn h2_multi_count() -> c_int;
    pub fn h2_msm_multi_gpu(curve: c_int, scalars: *const c_void, bases_xy: *const c_void, n: usize, repr: c_int, out_xyz: *mut c_void) -> c_int;
    pub fn h2_multi_bases_register(curve: c_int, bases_xy: *const c_void, n: usize, repr: c_int, handle: *mut u64) -> c_int;
    pub fn h2_multi_bases_release(handle: u64) -> c_int;
    pub fn h2_msm_multi_registered(handle: u64, scalars: *const c_void, n: usize, repr: c_int, out_xyz: *mut c_void) -> c_int;
    // prover lanes: one context per prover thread on the primary device
    pub fn h2_lane_create(lane: *mut u64) -> c_int;
    pub fn h2_lane_bind(lane: u64) -> c_int;
    pub fn h2_lane_destroy(lane: u64) -> c_int;
    // shared polynomials: one read-only proving key for every lane
    pub fn h2_poly_share(polys: *const u64, n: usize) -> c_int;
    pub fn h2_poly_permutation_product(z_out: *const u64, proofs: usize, columns: *const u64, sigmas: *const u64, cols: usize, chunk_len: u32,
                                       k: u32, beta: *const c_void, gamma: *const c_void, omega: *const c_void, delta: *const c_void,
                                       blinding: *const c_void, blinding_factors: u32, repr: c_int) -> c_int;
    pub fn h2_poly_lookup_product(z_out: *const u64, count: usize, inputs: *const u64, tables: *const u64, permuted_inputs: *const u64,
                                  permuted_tables: *const u64, k: u32, beta: *const c_void, gamma: *const c_void, blinding: *const c_void,
                                  blinding_factors: u32, repr: c_int) -> c_int;
    pub fn h2_poly_lookup_permuted(out_inputs: *const u64, out_tables: *const u64, count: usize, inputs: *const u64, tables: *const u64, k: u32,
                                   blinding: *const c_void, blinding_factors: u32, repr: c_int) -> c_int;
    pub fn h2_poly_lagrange_to_coeff_batch(dst: *const u64, src: *const u64, count: usize, k: u32, omega_inv: *const c_void, divisor: *const c_void,
                                           repr: c_int) -> c_int;
    pub fn h2_poly_coeff_to_extended_batch(dst: *const u64, src: *const u64, count: usize, k: u32, ext_k: u32, zeta: *const c_void,
                                           ext_omega: *const c_void, repr: c_int) -> c_int;
    pub fn h2_poly_set_rows(polys: *const u64, count: usize, start: usize, rows: usize, values: *const c_void, repr: c_int) -> c_int;
}

fn check(rc: c_int) {
    if rc != 0 {
        // the reference panics on misuse (arithmetic.rs:144,205); keep that behaviour
        let msg = unsafe { CStr::from_ptr(h2_last_error()) }.to_string_lossy().into_owned();
        panic!("halo2_b200: {}", msg);
    }
}

/// Curves the engine accelerates.
pub trait B200Curve: CurveAffine {
    const CURVE_ID: c_int;
    const SCALAR_FIELD_ID: c_int;
}
impl B200Curve for pallas::Affine {
    const CURVE_ID: c_int = CURVE_PALLAS;
    const SCALAR_FIELD_ID: c_int = FIELD_FQ;
}
impl B200Curve for vesta::Affine {
    const CURVE_ID: c_int = CURVE_VESTA;
    const SCALAR_FIELD_ID: c_int = FIELD_FP;
}

fn scalars_to_bytes<F: PrimeField>(s: &[F]) -> Vec<u8> {
    let mut out = Vec::with_capacity(32 * s.len());
    for x in s {
        out.extend_from_slice(x.to_repr().as_ref());
    }
    out
}
fn bases_to_bytes<C: CurveAffine>(b: &[C]) -> Vec<u8> {
    let mut out = vec![0u8; 64 * b.len()];
    for (i, p) in b.iter().enumerate() {
        if let Some(c) = Option::<pasta_curves::arithmetic::Coordinates<C>>::from(p.coordinates()) {
            out[64 * i..64 * i + 32].copy_from_slice(c.x().to_repr().as_ref());
            out[64 * i + 32..64 * i + 64].copy_from_slice(c.y().to_repr().as_ref());
        } // identity stays (0, 0)
    }
    out
}
fn point_from_xyz<C: B200Curve>(xyz: &[u8; 96]) -> C::Curve
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    let f = |o: usize| {
        let mut r = [0u8; 32];
        r.copy_from_slice(&xyz[o..o + 32]);
        C::Base::from_repr(r).unwrap()
    };
    C::CurveExt::new_jacobian(f(0), f(32), f(64)).unwrap().into()
}

/// Drop-in for `halo2_proofs::arithmetic::best_multiexp` (arithmetic.rs:143-180).
pub fn best_multiexp<C: B200Curve>(coeffs: &[C::Scalar], bases: &[C]) -> C::Curve
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    assert_eq!(coeffs.len(), bases.len());
    let s = scalars_to_bytes(coeffs);
    let b = bases_to_bytes(bases);
    let mut out = [0u8; 96];
    check(unsafe {
        h2_msm(C::CURVE_ID, s.as_ptr() as *const c_void, b.as_ptr() as *const c_void, coeffs.len(), REPR_CANONICAL,
               out.as_mut_ptr() as *mut c_void)
    });
    point_from_xyz::<C>(&out)
}

/// Drop-in for `best_fft` with G = Scalar (arithmetic.rs:192-255).
pub fn best_fft<F: PrimeField<Repr = [u8; 32]>>(field_id: c_int, a: &mut [F], omega: F, log_n: u32) {
    assert_eq!(a.len(), 1 << log_n);
    let mut bytes = scalars_to_bytes(a);
    let w = omega.to_repr();
    check(unsafe { h2_ntt(field_id, bytes.as_mut_ptr() as *mut c_void, w.as_ptr() as *const c_void, log_n, REPR_CANONICAL) });
    for (i, x) in a.iter_mut().enumerate() {
        let mut r = [0u8; 32];
        r.copy_from_slice(&bytes[32 * i..32 * i + 32]);
        *x = F::from_repr(r).unwrap();
    }
}

fn affine_from_xy<C: B200Curve>(xy: &[u8]) -> C
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    if xy.iter().all(|b| *b == 0) {
        return C::identity();
    }
    let f = |o: usize| {
        let mut r = [0u8; 32];
        r.copy_from_slice(&xy[o..o + 32]);
        C::Base::from_repr(r).unwrap()
    };
    C::from_xy(f(0), f(32)).unwrap()
}
fn curves_to_bytes<C: B200Curve>(pts: &[C::Curve]) -> Vec<u8>
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    let mut out = vec![0u8; 96 * pts.len()];
    for (i, p) in pts.iter().enumerate() {
        let (x, y, z) = p.jacobian_coordinates();
        out[96 * i..96 * i + 32].copy_from_slice(x.to_repr().as_ref());
        out[96 * i + 32..96 * i + 64].copy_from_slice(y.to_repr().as_ref());
        out[96 * i + 64..96 * i + 96].copy_from_slice(z.to_repr().as_ref());
    }
    out
}

/// Drop-in for `best_fft` with G = C::Curve (arithmetic.rs:192-255 through FftGroup, :17-27; Params::new,
/// poly/commitment.rs:81-82).
pub fn best_fft_curve<C: B200Curve>(a: &mut [C::Curve], omega: C::Scalar, log_n: u32)
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    assert_eq!(a.len(), 1 << log_n);
    let mut bytes = curves_to_bytes::<C>(a);
    let w = omega.to_repr();
    check(unsafe {
        h2_ec_fft(C::CURVE_ID, bytes.as_mut_ptr() as *mut c_void, w.as_ref().as_ptr() as *const c_void, log_n, std::ptr::null(), REPR_CANONICAL)
    });
    for (i, p) in a.iter_mut().enumerate() {
        let mut r = [0u8; 96];
        r.copy_from_slice(&bytes[96 * i..96 * i + 96]);
        *p = point_from_xyz::<C>(&r);
    }
}

/// Drop-in for `C::Curve::batch_normalize` (plonk/prover.rs:99,311; poly/commitment.rs:65,95).
pub fn batch_normalize<C: B200Curve>(p: &[C::Curve], q: &mut [C])
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    assert_eq!(p.len(), q.len());
    let bytes = curves_to_bytes::<C>(p);
    let mut out = vec![0u8; 64 * p.len()];
    check(unsafe { h2_batch_normalize(C::CURVE_ID, bytes.as_ptr() as *const c_void, p.len(), REPR_CANONICAL, out.as_mut_ptr() as *mut c_void) });
    for (i, a) in q.iter_mut().enumerate() {
        *a = affine_from_xy::<C>(&out[64 * i..64 * i + 64]);
    }
}

/// The `g -> g_lagrange` derivation of `Params::new` (poly/commitment.rs:74-101): alpha_inv and minv are the values
/// computed at :77-80 and :83.
pub fn params_lagrange<C: B200Curve>(g: &[C], k: u32, alpha_inv: C::Scalar, minv: C::Scalar) -> Vec<C>
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    assert_eq!(g.len(), 1 << k);
    let b = bases_to_bytes(g);
    let mut out = vec![0u8; 64 * g.len()];
    check(unsafe {
        h2_params_lagrange(C::CURVE_ID, b.as_ptr() as *const c_void, k, alpha_inv.to_repr().as_ref().as_ptr() as *const c_void,
                           minv.to_repr().as_ref().as_ptr() as *const c_void, REPR_CANONICAL, out.as_mut_ptr() as *mut c_void)
    });
    (0..g.len()).map(|i| affine_from_xy::<C>(&out[64 * i..64 * i + 64])).collect()
}

/// Postfix form of `poly::Ast` for `h2_poly_eval_ast` (halo2_b200/csrc/asteval.cuh).  The patched `Evaluator::evaluate`
/// (poly/evaluator.rs:129-228) calls `flatten(&ast, stride, &mut prog)` once and launches one kernel, instead of `recurse`
/// per chunk.  `AstView` is the shim's read-only mirror of the crate-private `Ast` enum (the patch adds the `From` impl
/// next to the enum, evaluator.rs:237-270).
pub enum AstView<'a, F> {
    Poly { index: usize, rotation: i32 },
    Add(&'a AstView<'a, F>, &'a AstView<'a, F>),
    Mul(&'a AstView<'a, F>, &'a AstView<'a, F>),
    Scale(&'a AstView<'a, F>, F),
    DistributePowers(&'a [AstView<'a, F>], F),
    LinearTerm(F),
    ConstantTerm(F),
}
#[derive(Default)]
pub struct AstProgram<F> {
    pub code: Vec<[u32; 4]>, // {op, arg, shift, 0}: 0 POLY 1 CONST 2 LINEAR 3 ADD 4 MUL 5 SCALE 6 NEG
    pub consts: Vec<F>,
}
impl<F: PrimeField> AstProgram<F> {
    fn konst(&mut self, v: F) -> u32 {
        if let Some(i) = self.consts.iter().position(|c| *c == v) {
            return i as u32;
        }
        self.consts.push(v);
        (self.consts.len() - 1) as u32
    }
    /// `stride` = 1 in the Lagrange basis, 2^(extended_k - k) in the extended one (poly/domain.rs:286-295).
    pub fn flatten(&mut self, ast: &AstView<'_, F>, stride: i32) {
        match ast {
            AstView::Poly { index, rotation } => self.code.push([0, *index as u32, (rotation * stride) as u32, 0]),
            AstView::Add(a, b) => { self.flatten(a, stride); self.flatten(b, stride); self.code.push([3, 0, 0, 0]); }
            AstView::Mul(a, b) => { self.flatten(a, stride); self.flatten(b, stride); self.code.push([4, 0, 0, 0]); }
            AstView::Scale(a, s) => { self.flatten(a, stride); let c = self.konst(*s); self.code.push([5, c, 0, 0]); }
            AstView::DistributePowers(terms, base) => {
                // fold from zero: acc = acc * base + term (evaluator.rs:182-193)
                let z = self.konst(F::ZERO);
                self.code.push([1, z, 0, 0]);
                for t in terms.iter() {
                    let b = self.konst(*base);
                    self.code.push([5, b, 0, 0]);
                    self.flatten(t, stride);
                    self.code.push([3, 0, 0, 0]);
                }
            }
            AstView::LinearTerm(s) => { let c = self.konst(*s); self.code.push([2, c, 0, 0]); }
            AstView::ConstantTerm(s) => { let c = self.konst(*s); self.code.push([1, c, 0, 0]); }
        }
    }
}

/// Bulk `C::from_bytes` for `Params::read` (poly/commitment.rs:183-205): `Err` where `C::read` would return `io::Error`.
pub fn read_points<C: B200Curve>(bytes: &[u8]) -> std::io::Result<Vec<C>>
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    assert_eq!(bytes.len() % 32, 0);
    let n = bytes.len() / 32;
    let mut out = vec![0u8; 64 * n];
    let rc = unsafe { h2_points_decompress(C::CURVE_ID, bytes.as_ptr() as *const c_void, n, REPR_CANONICAL, out.as_mut_ptr() as *mut c_void) };
    if rc != 0 {
        let msg = unsafe { CStr::from_ptr(h2_last_error()) }.to_string_lossy().into_owned();
        return Err(std::io::Error::new(std::io::ErrorKind::Other, msg));
    }
    Ok((0..n).map(|i| affine_from_xy::<C>(&out[64 * i..64 * i + 64])).collect())
}

/// Bulk `C::to_bytes` for `Params::write` (poly/commitment.rs:168-181).
pub fn write_points<C: B200Curve>(points: &[C]) -> Vec<u8> {
    let b = bases_to_bytes(points);
    let mut out = vec![0u8; 32 * points.len()];
    check(unsafe { h2_points_compress(C::CURVE_ID, b.as_ptr() as *const c_void, points.len(), REPR_CANONICAL, out.as_mut_ptr() as *mut c_void) });
    out
}

/// Resident generator set for `Params::{commit, commit_lagrange}` (poly/commitment.rs:119-150):
/// register `g ++ [w]` / `g_lagrange ++ [w]` once per `Params`, then each commit ships only the polynomial.
pub struct ResidentBases<C: B200Curve> {
    handle: u64,
    n: usize,
    _c: std::marker::PhantomData<C>,
}
impl<C: B200Curve> ResidentBases<C>
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    /// `bases` = g ++ [w] (commit only) or g ++ [w, u] (commit + IPA rounds).  The window table
    /// (H2_BASES_PRECOMPUTE = 1) makes every later MSM against this set a fixed-base one.
    pub fn new(bases: &[C]) -> Self {
        let b = bases_to_bytes(bases);
        let mut handle = 0u64;
        check(unsafe { h2_bases_register_ex(C::CURVE_ID, b.as_ptr() as *const c_void, bases.len(), REPR_CANONICAL, 0, 1, &mut handle) });
        Self { handle, n: bases.len(), _c: Default::default() }
    }
    /// [commit(p, r)] for several polynomials in one pass (plonk/prover.rs:305-309, vanishing/prover.rs:102-106).
    pub fn commit_many(&self, polys: &[&[C::Scalar]], blinds: &[C::Scalar]) -> Vec<C::Curve> {
        assert_eq!(polys.len(), blinds.len());
        let n = polys[0].len();
        let mut s = Vec::with_capacity(polys.len() * n * 32);
        for p in polys { assert_eq!(p.len(), n); s.extend_from_slice(&scalars_to_bytes(p)); }
        let r = scalars_to_bytes(blinds);
        let mut out = vec![0u8; 96 * polys.len()];
        check(unsafe {
            h2_msm_registered_batch(self.handle, s.as_ptr() as *const c_void, n, r.as_ptr() as *const c_void, polys.len(),
                                    REPR_CANONICAL, out.as_mut_ptr() as *mut c_void)
        });
        out.chunks(96).map(|c| point_from_xyz::<C>(c.try_into().unwrap())).collect()
    }
    /// The round loop of commitment::create_proof (poly/commitment/prover.rs:100-142).  `round` receives (L_j, R_j)
    /// and returns the challenge u_j (the caller's transcript); returns c = p_prime[0] after the last fold.
    pub fn ipa_rounds(&self, k: u32, p_prime: &[C::Scalar], x3: C::Scalar, z: C::Scalar,
                      mut rand: impl FnMut() -> (C::Scalar, C::Scalar),
                      mut round: impl FnMut(C::Curve, C::Curve, C::Scalar, C::Scalar) -> C::Scalar) -> C::Scalar {
        assert_eq!(self.n, (1usize << k) + 2);
        let pp = scalars_to_bytes(p_prime);
        let mut sess = 0u64;
        check(unsafe { h2_ipa_begin(self.handle, k, pp.as_ptr() as *const c_void, x3.to_repr().as_ref().as_ptr() as *const c_void,
                                    REPR_CANONICAL, &mut sess) });
        let zb = z.to_repr();
        for _ in 0..k {
            let (l_rand, r_rand) = rand();
            let mut lr = [0u8; 192];
            check(unsafe { h2_ipa_round(sess, zb.as_ref().as_ptr() as *const c_void, l_rand.to_repr().as_ref().as_ptr() as *const c_void,
                                        r_rand.to_repr().as_ref().as_ptr() as *const c_void, REPR_CANONICAL, lr.as_mut_ptr() as *mut c_void) });
            let l_j = point_from_xyz::<C>(lr[..96].try_into().unwrap());
            let r_j = point_from_xyz::<C>(lr[96..].try_into().unwrap());
            let u_j = round(l_j, r_j, l_rand, r_rand);
            let u_inv = u_j.invert().unwrap();
            check(unsafe { h2_ipa_fold(sess, u_j.to_repr().as_ref().as_ptr() as *const c_void,
                                       u_inv.to_repr().as_ref().as_ptr() as *const c_void, REPR_CANONICAL) });
        }
        let mut cb = [0u8; 64];
        check(unsafe { h2_ipa_finish(sess, REPR_CANONICAL, cb.as_mut_ptr() as *mut c_void) });
        let mut repr = <C::Scalar as PrimeField>::Repr::default();
        repr.as_mut().copy_from_slice(&cb[..32]);
        C::Scalar::from_repr(repr).unwrap()
    }
    /// <poly, bases[..n]> + r * bases[n]
    pub fn commit(&self, poly: &[C::Scalar], r: C::Scalar) -> C::Curve {
        assert!(poly.len() + 1 <= self.n);   // the blind rides on bases[poly.len()]; an IPA-capable set also holds u behind w
        let s = scalars_to_bytes(poly);
        let rb = r.to_repr();
        let mut out = [0u8; 96];
        check(unsafe {
            h2_msm_registered(self.handle, s.as_ptr() as *const c_void, poly.len(), rb.as_ref().as_ptr() as *const c_void,
                              REPR_CANONICAL, out.as_mut_ptr() as *mut c_void)
        });
        point_from_xyz::<C>(&out)
    }
}
impl<C: B200Curve> Drop for ResidentBases<C> {
    fn drop(&mut self) {
        unsafe { h2_bases_release(self.handle) };
    }
}

/// Call once per process (one process per GPU).
pub fn init(device: i32) {
    check(unsafe { h2_init(device) });
}

/// A prover lane bound to the current thread: every engine call this thread makes while the guard lives runs on a context
/// of its own (streams, scratch, caches, settings, resident polynomials and IPA sessions), concurrently with threads on other
/// lanes.  `ResidentBases` are shared by all lanes; resident polynomials (`h2_poly_*`) and IPA sessions belong to the lane
/// they were created on and are freed with it, except polynomials passed to `share_polys`.  Dropping the guard destroys the
/// lane and puts the thread back on the primary context.
/// Binding is per thread, so the guard is `!Send`.
pub struct Lane {
    handle: u64,
    _not_send: std::marker::PhantomData<*const ()>,
}
impl Lane {
    /// Creates a lane and binds the calling thread to it (after `init`; at most 16 lanes).
    pub fn new() -> Self {
        let mut handle = 0u64;
        check(unsafe { h2_lane_create(&mut handle) });
        if unsafe { h2_lane_bind(handle) } != 0 {
            unsafe { h2_lane_destroy(handle) };
            check(1);
        }
        Self { handle, _not_send: Default::default() }
    }
}
impl Drop for Lane {
    fn drop(&mut self) {
        unsafe { h2_lane_destroy(self.handle) };
    }
}

/// Shares resident polynomials of the calling thread's lane (or of the primary context) read-only with every lane and the
/// primary context (`h2_poly_share`): a proving key built once, on one lane, and read by the provers on all of them.  All or
/// nothing: every handle must be the caller's or already shared, else the call panics and nothing is shared.  Handles do not
/// change.  A shared handle may be used from any thread -- wherever a polynomial is only read, and by `h2_poly_free`, which
/// waits for the reads in progress on every lane -- so a key of shared handles can be `Send + Sync`.  An entry point that
/// would write a shared polynomial fails with a message saying it is shared; the lane that shared it may be dropped first.
pub fn share_polys(handles: &[u64]) {
    check(unsafe { h2_poly_share(handles.as_ptr(), handles.len()) });
}

/// One process, several GPUs: after `init(primary)`, bind `ngpu` devices; `best_multiexp_multi_gpu` then shards every call
/// (contiguous ranges, a 96-byte partial per device written to the primary over NVLink, one sum there).
pub fn multi_init(ngpu: i32) {
    check(unsafe { h2_multi_init(ngpu) });
}
/// `best_multiexp` (arithmetic.rs:143-180) over every device bound by `multi_init`.
pub fn best_multiexp_multi_gpu<C: B200Curve>(coeffs: &[C::Scalar], bases: &[C]) -> C::Curve {
    assert_eq!(coeffs.len(), bases.len());
    let (s, b) = (scalars_to_bytes(coeffs), bases_to_bytes(bases));
    let mut out = [0u8; 96];
    check(unsafe {
        h2_msm_multi_gpu(C::CURVE_ID, s.as_ptr() as *const c_void, b.as_ptr() as *const c_void, coeffs.len(), REPR_CANONICAL,
                         out.as_mut_ptr() as *mut c_void)
    });
    point_from_xyz::<C>(&out)
}

/// `permute_expression_pair` (plonk/lookup/prover.rs:563-647) on two resident Lagrange columns (handles from `h2_poly_alloc`):
/// the usable rows of `out_input` / `out_table` are written; the caller appends its random blinding rows (:625-627).
/// Returns false where the reference returns `Error::ConstraintSystemFailure` (:605-608).
pub fn lookup_permute_resident(input: u64, table: u64, usable_rows: usize, out_input: u64, out_table: u64) -> bool {
    unsafe { h2_poly_lookup_permute(input, table, usable_rows, out_input, out_table) == 0 }
}

/// The permutation polynomials of `Assembly::build_vk` / `build_pk` (plonk/permutation/keygen.rs:108-143, :161-198) as
/// resident Lagrange columns, built on the device without the n-element `omega_powers` / `deltaomega` tables.  `mapping` is
/// the reference's `Assembly::mapping` (one `Vec` of n = 2^k (column, row) pairs per permutation column), `omega` =
/// `domain.get_omega()`, `delta` = `F::DELTA`.  Returns one polynomial handle per column, owned by the caller's lane: commit
/// them (`h2_msm_registered_polys_affine`), transform them, and free them with `h2_poly_free`.  Panics on an out-of-range entry.
pub fn permutation_polys<F: PrimeField>(field_id: c_int, k: u32, mapping: &[Vec<(usize, usize)>], omega: F, delta: F) -> Vec<u64> {
    let n = 1usize << k;
    let mut flat = Vec::with_capacity(2 * n * mapping.len());
    for col in mapping {
        assert_eq!(col.len(), n);
        for &(c, r) in col {
            flat.push(u32::try_from(c).expect("column index >= 2^32"));
            flat.push(u32::try_from(r).expect("row index >= 2^32"));
        }
    }
    let mut handles = Vec::with_capacity(mapping.len());
    for _ in mapping {
        let mut h = 0u64;
        let rc = unsafe { h2_poly_alloc(field_id, n, &mut h) };
        if rc != 0 {
            for h in handles { unsafe { h2_poly_free(h) }; }
            check(rc);
        }
        handles.push(h);
    }
    let (w, d) = (omega.to_repr(), delta.to_repr());
    let rc = unsafe {
        h2_poly_permutation_sigma(handles.as_ptr(), handles.len(), k, flat.as_ptr(), w.as_ref().as_ptr() as *const c_void,
                                  d.as_ref().as_ptr() as *const c_void, REPR_CANONICAL)
    };
    if rc != 0 {
        for &h in &handles { unsafe { h2_poly_free(h) }; }
        check(rc);
    }
    handles
}

/// `permutation_polys` from the copy constraints themselves: `copies` holds one `[left column, left row, right column,
/// right row]` per `Assembly::copy` call, in synthesis order, columns as indices into the permutation's column list (what
/// `Assembly::copy` records after its own checks).  The cycles of `Assembly::mapping` are computed on the device, so no
/// mapping is built on the host.  Returns one polynomial handle per column, owned by the caller's lane.  Panics on a copy
/// out of range; the message names the first bad copy.
pub fn permutation_polys_from_copies<F: PrimeField>(field_id: c_int, k: u32, cols: usize, copies: &[[u32; 4]], omega: F, delta: F) -> Vec<u64> {
    let n = 1usize << k;
    let mut handles = Vec::with_capacity(cols);
    for _ in 0..cols {
        let mut h = 0u64;
        let rc = unsafe { h2_poly_alloc(field_id, n, &mut h) };
        if rc != 0 {
            for h in handles { unsafe { h2_poly_free(h) }; }
            check(rc);
        }
        handles.push(h);
    }
    let (w, d) = (omega.to_repr(), delta.to_repr());
    let rc = unsafe {
        h2_poly_permutation_sigma_copies(handles.as_ptr(), handles.len(), k, copies.as_ptr() as *const u32, copies.len(),
                                         w.as_ref().as_ptr() as *const c_void, d.as_ref().as_ptr() as *const c_void, REPR_CANONICAL)
    };
    if rc != 0 {
        for &h in &handles { unsafe { h2_poly_free(h) }; }
        check(rc);
    }
    handles
}

/// `count` zero-filled polynomials of n elements on the caller's lane; on a failure the ones already made are freed.
fn alloc_polys(field_id: c_int, n: usize, count: usize) -> Vec<u64> {
    let mut handles = Vec::with_capacity(count);
    for _ in 0..count {
        let mut h = 0u64;
        let rc = unsafe { h2_poly_alloc(field_id, n, &mut h) };
        if rc != 0 {
            for h in handles { unsafe { h2_poly_free(h) }; }
            check(rc);
        }
        handles.push(h);
    }
    handles
}

/// The permutation argument's product columns, `permutation::Argument::commit` (plonk/permutation/prover.rs:98-168) for every
/// proof at once: `columns` holds proof p's Lagrange columns at `[p * cols, (p + 1) * cols)` (advice, fixed or instance handles,
/// in the argument's column order), `sigmas` the key's `cols` permutation polynomials (a shared key works on every lane).
/// `blinding` holds `blinding_factors` values per (proof, set), in the rng's order.  Returns the z handles (Lagrange basis), set
/// after set and proof after proof, owned by the caller's lane; the call is asynchronous.  Commit them, then transform them.
pub fn permutation_products<F: PrimeField>(field_id: c_int, k: u32, columns: &[u64], sigmas: &[u64], chunk_len: u32, beta: F, gamma: F,
                                           omega: F, delta: F, blinding: &[F], blinding_factors: u32) -> Vec<u64> {
    assert!(!sigmas.is_empty() && chunk_len > 0 && columns.len() % sigmas.len() == 0, "one column per permutation polynomial and proof");
    let proofs = columns.len() / sigmas.len();
    let sets = (sigmas.len() + chunk_len as usize - 1) / chunk_len as usize;
    assert_eq!(blinding.len(), proofs * sets * blinding_factors as usize, "blinding_factors values per (proof, set)");
    let handles = alloc_polys(field_id, 1usize << k, proofs * sets);
    let (b, g, w, d, bl) = (beta.to_repr(), gamma.to_repr(), omega.to_repr(), delta.to_repr(), scalars_to_bytes(blinding));
    let rc = unsafe {
        h2_poly_permutation_product(handles.as_ptr(), proofs, columns.as_ptr(), sigmas.as_ptr(), sigmas.len(), chunk_len, k,
                                    b.as_ref().as_ptr() as *const c_void, g.as_ref().as_ptr() as *const c_void, w.as_ref().as_ptr() as *const c_void,
                                    d.as_ref().as_ptr() as *const c_void, bl.as_ptr() as *const c_void, blinding_factors, REPR_CANONICAL)
    };
    if rc != 0 {
        for &h in &handles { unsafe { h2_poly_free(h) }; }
        check(rc);
    }
    handles
}

/// The lookup argument's product columns, `lookup::Permuted::commit_product` (plonk/lookup/prover.rs:279-337), for every lookup
/// of every proof at once: entry b of the four slices is lookup b's compressed input, compressed table, permuted input and
/// permuted table (Lagrange handles).  `blinding` holds `blinding_factors` values per lookup.  Returns the z handles
/// (Lagrange basis), owned by the caller's lane; the call is asynchronous.
pub fn lookup_products<F: PrimeField>(field_id: c_int, k: u32, inputs: &[u64], tables: &[u64], permuted_inputs: &[u64], permuted_tables: &[u64],
                                      beta: F, gamma: F, blinding: &[F], blinding_factors: u32) -> Vec<u64> {
    let count = inputs.len();
    assert!(tables.len() == count && permuted_inputs.len() == count && permuted_tables.len() == count, "four columns per lookup");
    assert_eq!(blinding.len(), count * blinding_factors as usize, "blinding_factors values per lookup");
    let handles = alloc_polys(field_id, 1usize << k, count);
    let (b, g, bl) = (beta.to_repr(), gamma.to_repr(), scalars_to_bytes(blinding));
    let rc = unsafe {
        h2_poly_lookup_product(handles.as_ptr(), count, inputs.as_ptr(), tables.as_ptr(), permuted_inputs.as_ptr(), permuted_tables.as_ptr(), k,
                               b.as_ref().as_ptr() as *const c_void, g.as_ref().as_ptr() as *const c_void, bl.as_ptr() as *const c_void,
                               blinding_factors, REPR_CANONICAL)
    };
    if rc != 0 {
        for &h in &handles { unsafe { h2_poly_free(h) }; }
        check(rc);
    }
    handles
}

/// The permuted columns of `commit_permuted` (plonk/lookup/prover.rs:76-243) for every lookup of every proof in one call:
/// `inputs[b]` / `tables[b]` are lookup b's compressed Lagrange columns (handles, 2^k elements; shared ones work on every
/// lane), `blinding` holds per lookup blinding_factors + 1 input rows then as many table rows, in the rng's order
/// (:622-624).  Returns (permuted input, permuted table) handles per lookup, blinding rows included.  Panics, naming the lowest
/// lookup, where the reference returns Error::ConstraintSystemFailure (an input value missing from its table).
pub fn lookup_permuted<F: PrimeField>(field_id: c_int, k: u32, inputs: &[u64], tables: &[u64], blinding: &[F], blinding_factors: u32) -> Vec<(u64, u64)> {
    let count = inputs.len();
    assert_eq!(tables.len(), count, "one table per input");
    assert_eq!(blinding.len(), count * 2 * (blinding_factors as usize + 1), "2 (blinding_factors + 1) values per lookup");
    let outs = alloc_polys(field_id, 1usize << k, 2 * count);
    let (oi, ot): (Vec<u64>, Vec<u64>) = (outs[..count].to_vec(), outs[count..].to_vec());
    let bl = scalars_to_bytes(blinding);
    let rc = unsafe {
        h2_poly_lookup_permuted(oi.as_ptr(), ot.as_ptr(), count, inputs.as_ptr(), tables.as_ptr(), k, bl.as_ptr() as *const c_void, blinding_factors,
                                REPR_CANONICAL)
    };
    if rc != 0 {
        for &h in &outs { unsafe { h2_poly_free(h) }; }
        check(rc);
    }
    oi.into_iter().zip(ot).collect()
}

/// The verifier's `g_scalars` (poly/commitment/msm.rs:12) kept in HBM: what `MSM<C>` holds under the `b200` feature instead of
/// `Option<Vec<C::Scalar>>`.  `compute_s` (poly/commitment/verifier.rs:156-171) is built on the device straight into it,
/// `scale` / `add_msm` (msm.rs:37-62, :122-135) are one elementwise pass, and `eval` (msm.rs:138-177) commits the resident vector
/// against the resident generators (`w_scalar` rides on base index n) and adds the multiexp of the few dozen other terms.
pub struct ResidentGScalars<C: B200Curve> {
    handle: u64,
    n: usize,
    _c: std::marker::PhantomData<C>,
}
impl<C: B200Curve> ResidentGScalars<C>
where
    C::Base: PrimeField<Repr = [u8; 32]>,
{
    /// `vec![C::Scalar::ZERO; params.n]` (msm.rs:91): zero-filled on the device.
    pub fn zeros(n: usize) -> Self {
        let mut handle = 0u64;
        check(unsafe { h2_poly_alloc(C::SCALAR_FIELD_ID, n, &mut handle) });
        ResidentGScalars { handle, n, _c: std::marker::PhantomData }
    }
    /// `g_scalars[0] += constant` (msm.rs:87-95).
    pub fn add_constant_term(&mut self, constant: C::Scalar) {
        check(unsafe { h2_poly_add_at(self.handle, 0, constant.to_repr().as_ref().as_ptr() as *const c_void, REPR_CANONICAL) });
    }
    /// `self.add_to_g_scalars(&compute_s(u, init))` (verifier.rs:36-38) in one pass; panics for an empty `u` like the reference (:157).
    pub fn add_compute_s(&mut self, u: &[C::Scalar], init: C::Scalar) {
        assert_eq!(1usize << u.len(), self.n);
        let ub = scalars_to_bytes(u);
        check(unsafe {
            h2_poly_compute_s(self.handle, ub.as_ptr() as *const c_void, u.len() as u32, init.to_repr().as_ref().as_ptr() as *const c_void,
                              1, REPR_CANONICAL)
        });
    }
    /// `g_scalar *= factor` for every entry (msm.rs:126-131).
    pub fn scale(&mut self, factor: C::Scalar) {
        check(unsafe {
            h2_poly_scale_add(self.handle, factor.to_repr().as_ref().as_ptr() as *const c_void, 0, std::ptr::null(), self.n, REPR_CANONICAL)
        });
    }
    /// `self = factor * self + other`: `acc.scale(r); acc.add_msm(&msm)` of BatchVerifier::finalize (plonk/verifier/batch.rs:83-93)
    /// for the vector part, one pass; `factor = 1` is the plain `add_to_g_scalars` of msm.rs:52-54.
    pub fn scale_add(&mut self, factor: C::Scalar, other: &Self) {
        assert_eq!(self.n, other.n);
        let one = C::Scalar::ONE.to_repr();
        check(unsafe {
            h2_poly_scale_add(self.handle, factor.to_repr().as_ref().as_ptr() as *const c_void, other.handle,
                              one.as_ref().as_ptr() as *const c_void, self.n, REPR_CANONICAL)
        });
    }
    /// The multiexp of `MSM::eval` (msm.rs:142-175): <g_scalars, g> + w_scalar * w over the resident set `g ++ [w, u]`, plus the
    /// other terms (`u`, the proof's commitments) through the plain MSM; the caller tests `is_identity()`.
    pub fn eval_with(&self, g: &ResidentBases<C>, w_scalar: C::Scalar, other_scalars: &[C::Scalar], other_bases: &[C]) -> C::Curve {
        let mut out = [0u8; 96];
        check(unsafe {
            h2_msm_registered_polys(g.handle, &self.handle as *const u64, 1, self.n, w_scalar.to_repr().as_ref().as_ptr() as *const c_void,
                                    REPR_CANONICAL, out.as_mut_ptr() as *mut c_void)
        });
        point_from_xyz::<C>(&out) + best_multiexp::<C>(other_scalars, other_bases)
    }
}
impl<C: B200Curve> Drop for ResidentGScalars<C> {
    fn drop(&mut self) {
        unsafe { h2_poly_free(self.handle) };
    }
}
