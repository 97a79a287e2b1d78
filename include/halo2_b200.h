/*
 * halo2_b200 -- C ABI of the H100-native MSM + NTT engine for the halo2 prover hot path.
 *
 * The reference (zcash/halo2, pure Rust) has no FFI: the boundary is four generic Rust
 * functions.  Each entry point below names the reference interface it replaces
 * (paths relative to /root/reference/halo2_proofs/src).  INTEGRATION.md shows the Rust
 * `halo2-b200-sys` binding and the patched arithmetic.rs dispatch a maintainer would add.
 *
 * Conventions
 *   - Plain pointers and sizes only.  All functions return 0 on success, non-zero on error;
 *     h2_last_error() gives the message (thread-local).  The Rust shim panics on non-zero,
 *     preserving the reference's assert!/panic! error behaviour (arithmetic.rs:144,205).
 *   - Field element = 32 bytes = 4 x u64 little-endian limbs.  `repr` selects the encoding:
 *       H2_REPR_CANONICAL   the integer itself (ff::PrimeField::to_repr, arithmetic.rs:77)
 *       H2_REPR_MONTGOMERY  x * 2^256 mod m (pasta_curves' in-memory form: zero-copy path)
 *     for every host element and point a call takes or returns (coordinate by coordinate).  Before it copies or
 *     launches anything, a call fails with "<entry point>: unknown repr" for any other value, and with
 *     "<entry point>: null <parameter>" when a host element or element array it reads or writes is NULL.  An array of
 *     no elements may be NULL, and so may an element the call does not touch: every element of a call with nothing
 *     to do (count, cols or proofs == 0), the init of a running product of n == 0, the points of an evaluation of
 *     n == 0 or of a Kate division of n <= 1; so may the optional pointers documented below.  repr is checked even then.
 *   - Affine point = x || y (64 bytes); the identity is 64 zero bytes
 *     (book/src/background/curves.md:226-230).  Results are Jacobian x || y || z (96 bytes,
 *     the layout of pasta's Ep/Eq); identity has z = 0.  Only the group element is defined
 *     (the reference compares with == on C::Curve, arithmetic.rs:457).
 *   - curve: H2_CURVE_PALLAS = EpAffine (coordinates Fp, scalars Fq),
 *            H2_CURVE_VESTA  = EqAffine (coordinates Fq, scalars Fp).
 *   - Thread-safe and re-entrant (BatchVerifier calls commit_lagrange from many rayon
 *     workers, plonk/verifier/batch.rs:97-110): calls on one context are serialised on its
 *     lock.  A thread that binds a lane (h2_lane_bind) gets a context of its own, so calls
 *     from threads on different lanes run concurrently on the GPU.
 *   - There is NO CPU fallback: every function fails if no CUDA device is usable.
 *   - Functions suffixed _dev take CUDA device pointers (Montgomery form) and a cudaStream_t
 *     (passed as void*); they do not synchronise.  The others take host pointers, copy in
 *     and out, and return when the result is in the caller's buffer.
 */
#ifndef HALO2_B200_H
#define HALO2_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { H2_CURVE_PALLAS = 0, H2_CURVE_VESTA = 1 };
enum { H2_FIELD_FP = 0, H2_FIELD_FQ = 1 };
enum { H2_REPR_CANONICAL = 0, H2_REPR_MONTGOMERY = 1 };

/* ---- lifecycle ------------------------------------------------------------------------- */
/* Binds the engine to CUDA device `device` (one process per GPU).  Idempotent. */
int h2_init(int device);
int h2_shutdown(void);
const char *h2_last_error(void);
int h2_device_count(void);
/* ABI version of this header (bumped on incompatible change). */
uint32_t h2_abi_version(void);

/* ---- lanes: independent provers on one GPU ------------------------------------------------------------------------
 * A lane is one more context on the primary device: its own streams, scratch pools, staging ring, twiddle and graph
 * caches and settings, and its own resident polynomials and IPA sessions.  A host thread bound to a lane runs every call
 * there, concurrently with the threads on other lanes; a thread that never binds uses the primary context.
 *   - h2_lane_create fails before h2_init and when all 16 lanes exist.  A new lane starts with the library's default
 *     settings; h2_set_window_bits / h2_set_glv / h2_set_sort_mode, the h2_test_set_* hooks except the process-wide
 *     staging, copy-thread and chunk-cut ones, and h2_test_last_msm_plan act on the calling thread's lane.
 *   - h2_lane_bind(0) goes back to the primary context.  Binding an unknown lane fails.
 *   - Polynomial and IPA-session handles belong to the lane that created them; from any other lane (the primary
 *     included) they are unknown, until h2_poly_share makes polynomials read-only and readable from every lane and the
 *     primary context (one proving key for all lanes).  Base sets (h2_bases_register*) are shared by every lane.
 *   - h2_lane_destroy frees the lane's polynomials (not those it shared), IPA sessions and pools; it fails while another thread is bound to
 *     the lane.  h2_shutdown destroys every lane; lane handles from before it are unknown afterwards, and a thread that
 *     was bound must bind again.
 *   - The h2_multi_* entry points fail on a thread bound to a lane. */
int h2_lane_create(uint64_t *lane);
int h2_lane_bind(uint64_t lane);
int h2_lane_destroy(uint64_t lane);

/* ---- MSM: replaces best_multiexp, arithmetic.rs:143-180 ------------------------------------ */
/* out = sum_i scalars[i] * bases[i].  Caller guarantees both arrays hold n entries
 * (the shim asserts coeffs.len() == bases.len() like arithmetic.rs:144). */
int h2_msm(int curve, const void *scalars, const void *bases_xy, size_t n, int repr, void *out_xyz);

/* Params::{g, g_lagrange} ++ [w] are immutable for the life of a Params (poly/commitment.rs:26-33):
 * upload once, commit many times.  Replaces the per-call Vec copies of commit/commit_lagrange
 * (poly/commitment.rs:119-150). */
int h2_bases_register(int curve, const void *bases_xy, size_t n, int repr, uint64_t *handle);
/* Same, with options.  flags & H2_BASES_PRECOMPUTE: also build the window table
 * T[w][i] = 2^(c w) * bases[i] (W = ceil(256/c) affine copies, c = window_bits or automatic when 0).
 * h2_msm_registered then drops every window's digits into ONE bucket set: no window combine, 1/W of
 * the bucket reduce -- what makes k = 14 sized commits latency-friendly. */
enum { H2_BASES_PRECOMPUTE = 1, H2_BASES_DIRECT = 2 };
/* flags & H2_BASES_DIRECT (with H2_BASES_PRECOMPUTE, sets of at most 2^15 + 2 points): also build the digit-multiples table
 * D[i][w][m] = m * 2^(8 w) * bases[i] (32 windows x 128 multiples, 256 KiB per point: 4.3 GB at k = 14).  Every fixed-base
 * MSM over the set -- commits, batches, IPA rounds -- is then a plain sum of the n x 32 entries the signed base-256 digits
 * select (three launches, no buckets): halo2_b200/csrc/fixedbase.cuh.  Same group element either way. */
int h2_bases_register_ex(int curve, const void *bases_xy, size_t n, int repr, uint32_t window_bits, uint32_t flags,
                         uint64_t *handle);
/* Base sets are shared by every lane.  Waits for calls on other lanes that are reading the set; fails while an open IPA
 * session on any lane refers to it (h2_ipa_finish first). */
int h2_bases_release(uint64_t handle);
/* sum_{i<n} scalars[i] * bases[i]  (+ extra_scalar[0] * bases[n] when extra_scalar != NULL):
 * commit(poly, r) = h2_msm_registered(h(g ++ [w]), poly, n, &r, ...). */
int h2_msm_registered(uint64_t handle, const void *scalars, size_t n, const void *extra_scalar, int repr,
                      void *out_xyz);

/* `batch` polynomials against the same resident table in ONE pass (bucket set = polynomial index):
 * the advice-column commits (plonk/prover.rs:305-309), the h(X) pieces (vanishing/prover.rs:102-106), ...
 * scalars: batch x n contiguous; extra_scalars: batch blinds or NULL; out_xyz: batch x 96 bytes.
 * Needs a base set registered with H2_BASES_PRECOMPUTE. */
int h2_msm_registered_batch(uint64_t handle, const void *scalars, size_t n, const void *extra_scalars, size_t batch, int repr,
                            void *out_xyz);
/* The same pass followed by C::Curve::batch_normalize on the device -- the shape of plonk/prover.rs:305-311 (commit
 * every advice column, then normalise the batch for the transcript): out_xy receives `batch` affine points (64 B). */
int h2_msm_registered_batch_affine(uint64_t handle, const void *scalars, size_t n, const void *extra_scalars, size_t batch, int repr,
                                   void *out_xy);

/* ---- IPA opening: the round loop of commitment::create_proof, poly/commitment/prover.rs:100-142 ----
 * Replaces, per round j: the two best_multiexp calls over the folded generators (:107-108), the two
 * compute_inner_product calls (:110-111), the [value z]U + [rand]W terms (:113-119), the folds of p' and b
 * (:134-139) and parallel_generator_collapse (:140, :154-166).  The generators are never folded on the device:
 * L_j and R_j are fixed-base MSMs over the resident table with the accumulated challenge products folded into
 * the scalars (halo2_b200/csrc/ipa.cuh) -- same group elements, same affine encodings.
 * The transcript (challenges) and the randomness stay with the caller:
 *
 *   h2_ipa_begin(h, k, p_prime, x3, repr, &s);           // p_prime: prover.rs:80, b = powers of x3: :86-93
 *   for j in 0..k {
 *       h2_ipa_round(s, z, l_rand_j, r_rand_j, repr, LR); // LR = L_j || R_j, 2 x 96 bytes (x, y, z), :107-119
 *       ... write to_affine(L_j), to_affine(R_j) to the transcript, squeeze u_j ...
 *       h2_ipa_fold(s, u_j, u_j_inv, repr);               // :134-140 (asynchronous)
 *   }
 *   h2_ipa_finish(s, repr, cb);                           // cb = c (= p_prime[0], :147) || b[0], 2 x 32 bytes
 *
 * `bases_handle` must be a set of 2^k + 2 points g[0..2^k) || w || u registered with H2_BASES_PRECOMPUTE
 * (the same set serves commit(): w sits at index n).  h2_ipa_finish with out_c_b == NULL aborts a session. */
int h2_ipa_begin(uint64_t bases_handle, uint32_t k, const void *p_prime, const void *x3, int repr, uint64_t *session);
/* p' taken from a device-resident polynomial (h2_poly_* handle, 2^k coefficients): nothing but x3 goes up. */
int h2_ipa_begin_poly(uint64_t bases_handle, uint32_t k, uint64_t p_prime_poly, const void *x3, int repr, uint64_t *session);
int h2_ipa_round(uint64_t session, const void *z, const void *l_rand, const void *r_rand, int repr, void *out_lr_xyz);
/* L_j, R_j as the two AFFINE points the prover writes to the transcript (`to_affine`, prover.rs:120-125): 2 x 64 B. */
int h2_ipa_round_affine(uint64_t session, const void *z, const void *l_rand, const void *r_rand, int repr, void *out_lr_xy);
int h2_ipa_fold(uint64_t session, const void *u, const void *u_inv, int repr);
int h2_ipa_finish(uint64_t session, int repr, void *out_c_b);

/* Window size override for the sweep in BASELINE.json config 3 (0 = automatic). */
int h2_set_window_bits(uint32_t c);
/* ---- Device-resident polynomials (SURVEY.md section 8(f) row 3: the quotient pipeline without a PCIe round trip per
 * call).  A polynomial lives in HBM in Montgomery form; the transforms below are the resident forms of
 * h2_intt_scaled / h2_coeff_to_extended / h2_extended_to_coeff (poly/domain.rs:227-255, :303-325) and are asynchronous
 * (stream-ordered); h2_msm_registered_polys is Params::commit / commit_lagrange (poly/commitment.rs:119-150) of `batch`
 * resident polynomials in one pass.  `repr` is the encoding of the host-side constants / blinds / results.
 *
 *   h2_poly_alloc(field, n, &v); h2_poly_upload(v, values, n, repr);          // Lagrange values, once
 *   h2_poly_lagrange_to_coeff(v, v, k, omega_inv, ifft_divisor, repr);        // in place
 *   h2_msm_registered_polys(params_g, &v, 1, n, &blind, repr, commitment);
 *   h2_poly_alloc(field, 4 n, &e); h2_poly_coeff_to_extended(e, v, k, k + 2, zeta, ext_omega, repr);
 *   h2_poly_download(e, evals, 4 n, repr);                                    // for the h(X) evaluation on the host
 */
int h2_poly_alloc(int field, size_t len, uint64_t *poly);
/* A polynomial of the calling context goes back to its pool.  A shared one (h2_poly_share) may be freed from any thread on
 * any lane or the primary context: no new call finds it, the calls in progress that read it finish, the device is
 * synchronised (asynchronous reads queued on any lane's stream) and the buffer is freed. */
int h2_poly_free(uint64_t poly);
/* Shares the calling context's polynomials polys[0 .. n) read-only with every lane and the primary context: a proving key
 * built once and read by every prover lane.  Each handle must be the calling context's or already shared (a no-op); any
 * other handle fails the call and then nothing is shared.  Synchronises the context's stream once, so every write to them
 * has landed.  Handles do not change.  A shared handle is accepted wherever a polynomial is only read (downloads, the
 * sources of copies, transforms, running products, Kate divisions and scale_add, the operands of eval_ast / eval /
 * inner_product, the inputs of lookup_permute and of the product columns, h2_msm_registered_polys*, h2_ipa_begin_poly); every call that would write
 * one fails with "<entry point>: the polynomial is shared (read-only)" and changes nothing.  Every rejected polynomial
 * handle is reported this way, "<entry point>: <reason>"; an element of a handle array as "<entry point>: <name>[i]:
 * <reason>", and an output that another argument also names as "<entry point>: dst[2] is also dst[0]".  h2_lane_destroy of the lane
 * that shared it leaves it alive; h2_shutdown frees every shared polynomial.  n == 0 does nothing; fails before h2_init. */
int h2_poly_share(const uint64_t *polys, size_t n);
int h2_poly_upload(uint64_t poly, const void *src, size_t len, int repr);
int h2_poly_download(uint64_t poly, void *dst, size_t len, int repr);
/* a[index] += delta on a resident polynomial: the one-coefficient corrections of the opening argument
 * (poly/commitment/prover.rs:51 `s_poly[0] -= s_at_x3`, :78 `p_prime_poly[0] -= v`). */
int h2_poly_add_at(uint64_t poly, size_t index, const void *delta, int repr);
/* dst[dst_off .. +len) = src[src_off .. +len) on the device: the h(X) pieces (plonk/vanishing/prover.rs:95-100,
 * `h_poly.chunks_exact(n)`), or a copy of a column that an in-place step is about to overwrite. */
int h2_poly_copy(uint64_t dst, size_t dst_off, uint64_t src, size_t src_off, size_t len);
int h2_poly_lagrange_to_coeff(uint64_t dst, uint64_t src, uint32_t k, const void *omega_inv, const void *divisor, int repr);
int h2_poly_coeff_to_extended(uint64_t dst, uint64_t src, uint32_t k, uint32_t ext_k, const void *zeta, const void *ext_omega, int repr);
int h2_poly_extended_to_coeff(uint64_t dst, uint64_t src, uint32_t ext_k, const void *ext_omega_inv, const void *ext_divisor,
                              const void *zeta, size_t out_len, int repr);
/* The same transforms for `count` columns of one size and domain in one call: dst[i] = lagrange_to_coeff(src[i]) /
 * coeff_to_extended(src[i]), the instance and advice phases of plonk::create_proof (plonk/prover.rs:79-124, :269-335).  Each
 * pass is one launch for the whole batch (the launches of one column, while count x 2^log_n x 32 B of scratch stays within
 * 256 MiB; larger batches run in groups of that size).  Sources are only read and may repeat, so shared polynomials work;
 * destinations must be the calling context's own, pairwise distinct and none of the other columns' sources.  dst[i] == src[i]
 * transforms column i in place where the one-column call allows it (equal input and output sizes).  Every check runs before
 * anything is launched and a failed call changes nothing; messages name the first offending index ("dst[3]").  count == 0
 * does nothing.  Asynchronous, like the one-column calls. */
int h2_poly_lagrange_to_coeff_batch(const uint64_t *dst, const uint64_t *src, size_t count, uint32_t k, const void *omega_inv,
                                    const void *divisor, int repr);
int h2_poly_coeff_to_extended_batch(const uint64_t *dst, const uint64_t *src, size_t count, uint32_t k, uint32_t ext_k, const void *zeta,
                                    const void *ext_omega, int repr);
/* Rows [start, start + rows) of each of `count` resident polynomials <- values (count x rows elements in `repr`, column by
 * column), one upload and one kernel: the blinding rows of advice columns that are already resident (plonk/prover.rs:276-282).
 * The polynomials must be the calling context's own and pairwise distinct, each with at least start + rows elements; every
 * check runs first and a failed call changes nothing.  count == 0 or rows == 0 does nothing.  Asynchronous. */
int h2_poly_set_rows(const uint64_t *polys, size_t count, size_t start, size_t rows, const void *values, int repr);
int h2_msm_registered_polys(uint64_t bases_handle, const uint64_t *polys, size_t batch, size_t n, const void *extra_scalars, int repr,
                            void *out_xyz);
/* The same pass followed by batch_normalize on the device: `batch` affine points (64 B each) -- what the prover writes to
 * the transcript (plonk/prover.rs:305-316 commit + batch_normalize + write_point). */
int h2_msm_registered_polys_affine(uint64_t bases_handle, const uint64_t *polys, size_t batch, size_t n, const void *extra_scalars,
                                   int repr, void *out_xy);

/* The prover's coefficient-form reductions on resident polynomials (SURVEY.md section 8(f) row 3), each a tree of
 * 32-coefficient serial pieces instead of the reference's serial loop; `batch` polynomials of n coefficients per call.
 * eval_polynomial (arithmetic.rs:297-303): out[i] = polys[i](points[i]); points / out are batch x 32 bytes on the host. */
int h2_poly_eval(const uint64_t *polys, size_t batch, size_t n, const void *points, int repr, void *out);
/* Evaluator::evaluate (poly/evaluator.rs:129-228) on resident polynomials of one basis: out[i] = Ast(polys)[i] for i < 2^log_n.
 * `code` is the postfix form of the Ast, n_code instructions of four uint32 {op, arg, shift, 0}:
 *   0 POLY   push polys[arg][(i + shift) mod 2^log_n]   (shift = rotation * stride; stride = 2^(extended_k - k) in the extended basis)
 *   1 CONST  push consts[arg]            2 LINEAR push consts[arg] * lin_base * omega^i   (lin_base = 1 | zeta, :538-555, :584-604)
 *   3 ADD    4 MUL  (two operands -> one)   5 SCALE top *= consts[arg]     6 NEG
 * (DistributePowers, :182-193, flattens to CONST 0, then SCALE base / term / ADD per term.)  The output cannot be an operand.
 * omega / lin_base may be NULL when the program has no LINEAR.  Asynchronous. */
int h2_poly_eval_ast(uint64_t out, const uint64_t *polys, size_t n_polys, uint32_t log_n, const uint32_t *code, size_t n_code,
                     const void *consts, size_t n_consts, const void *omega, const void *lin_base, int repr);
/* The permutation / lookup arguments' grand product (plonk/permutation/prover.rs:98-157) on resident polynomials:
 * `modified_values.batch_invert()` (ff::BatchInvert: in place, zeros stay zero) ... */
int h2_poly_batch_invert(uint64_t poly, size_t n);
/* ... and the running product dst[0] = init (last_z), dst[i] = dst[i - 1] * src[i - 1], i < n (:150-156).  The elementwise
 * numerators / denominators before it are Ast programs in the Lagrange basis (h2_poly_eval_ast).  Both asynchronous. */
int h2_poly_running_product(uint64_t dst, uint64_t src, size_t n, const void *init, int repr);
/* The lookup argument's permuted columns, permute_expression_pair (plonk/lookup/prover.rs:563-647), on resident Lagrange-basis
 * polynomials: out_input[0, usable_rows) = the input values sorted (ff's Ord = the canonical integers, :577-581);
 * out_table[r] = out_input[r] on the first row of every run of equal values (:595-603), the remaining rows take the table
 * values that are left over, ascending, from the last such row down (:617-622).  Rows from usable_rows on -- the blinding rows,
 * :625-627 -- are not touched: the caller writes its random values there.  Fails (non-zero, the outputs unchanged) when
 * an input value does not occur in the table, the reference's Error::ConstraintSystemFailure (:605-608).  Synchronous. */
int h2_poly_lookup_permute(uint64_t input, uint64_t table, size_t usable_rows, uint64_t out_input, uint64_t out_table);
/* The same permuted columns for `count` lookups (of any number of proofs) in one call, blinding rows included:
 * lookup::Argument::commit_permuted (plonk/lookup/prover.rs:76-243) between compressing the expressions and committing.
 * Every lookup has n = 2^k rows and u = n - blinding_factors - 1 usable ones: out_inputs[b] / out_tables[b] rows [0, u) =
 * permute_expression_pair of inputs[b] / tables[b] as h2_poly_lookup_permute gives them, rows [u, n) = the caller's random
 * values.  blinding: count x 2 (blinding_factors + 1) elements in `repr`, per lookup the input's rows then the table's, the
 * reference's rng order (:622-624).  The inputs are only read and may repeat, so shared polynomials work on every lane; the
 * outputs must be the calling context's own, pairwise distinct and none of the inputs.  Every check runs before anything is
 * launched, and a failed check writes nothing: unknown handle, other field, fewer than n elements, shared output, aliasing,
 * blinding_factors + 1 >= n, k > 30, count > 65535.  When an input value does not occur in its table
 * (Error::ConstraintSystemFailure, :605-608) the call fails naming the lowest such lookup b, and no output has changed.
 * count == 0 does nothing.  Synchronous: one synchronisation whatever count is. */
int h2_poly_lookup_permuted(const uint64_t *out_inputs, const uint64_t *out_tables, size_t count, const uint64_t *inputs,
                            const uint64_t *tables, uint32_t k, const void *blinding, uint32_t blinding_factors, int repr);
/* EvaluationDomain::divide_by_vanishing_poly (poly/domain.rs:329-348) in place on a resident extended-domain polynomial:
 * h[i] *= t_evals[i mod t_len]; t_evals = the domain's t_evaluations (domain.rs:86-128), t_len = 2^(ext_k - k).  Asynchronous. */
int h2_poly_divide_by_vanishing(uint64_t poly, uint32_t ext_k, const void *t_evals, uint32_t t_len, int repr);
/* The vanishing argument's quotient h(X) in pieces (plonk/vanishing/prover.rs:84-100): pieces[i] <- coefficients
 * [i 2^k, (i + 1) 2^k) of extended_to_coeff(divide_by_vanishing_poly(src)), i < count, in one transform of 2^ext_k points.
 * The division by t(X) = X^n - 1 is fused into the first NTT pass, the zeta un-shift, the 1 / 2^ext_k scaling and the split
 * into the last; the bytes equal h2_poly_divide_by_vanishing + h2_poly_extended_to_coeff + count h2_poly_copy calls.  src
 * (2^ext_k extended-domain evaluations) is only read and may be shared; the pieces must be the calling context's own, hold
 * 2^k elements each, be pairwise distinct and not src.  Requires k <= ext_k <= 30, 1 <= count <= 2^(ext_k - k) and t_len a
 * power of two <= 2^ext_k (t_evals as for h2_poly_divide_by_vanishing).  Every check runs before anything is launched, a
 * failed call changes nothing, and messages name the argument and index ("pieces[2]").  Asynchronous. */
int h2_poly_vanishing_quotient(const uint64_t *pieces, size_t count, uint64_t src, uint32_t k, uint32_t ext_k, const void *ext_omega_inv,
                               const void *ext_divisor, const void *zeta, const void *t_evals, uint32_t t_len, int repr);
/* compute_inner_product (arithmetic.rs:308-319): out[i] = sum_j a[i][j] * b[i][j]. */
int h2_poly_inner_product(const uint64_t *a, const uint64_t *b, size_t batch, size_t n, int repr, void *out);
/* kate_division (arithmetic.rs:322-341): dst[i] <- the n - 1 coefficients of (src[i] - src[i](points[i])) / (X - points[i]);
 * dst[i] must be a different polynomial with room for n - 1 coefficients.  Asynchronous. */
int h2_poly_kate_division(const uint64_t *dst, const uint64_t *src, size_t batch, size_t n, const void *points, int repr);

/* ---- The verifier's side: MSM<C> (poly/commitment/msm.rs:9-178) with its g_scalars vector resident -------------------------
 * The verifier's hot path is MSM::eval (msm.rs:142-177): ONE best_multiexp over params.g (2^k resident bases) plus w, u and
 * the few dozen commitments of the proof.  Its g_scalars is a polynomial handle of the curve's scalar field; `other`, w_scalar
 * and u_scalar stay with the caller (a few dozen scalars).  eval = h2_msm_registered_polys over the resident g (w_scalar rides
 * on base index n) + h2_msm over the other terms + h2_point_sum, identity <=> z = 0.
 *
 * compute_s (poly/commitment/verifier.rs:156-171): dst[i] = init * prod_{j : bit j of i} u[k - 1 - j] for i < 2^k, u = the
 * k round challenges u_0 .. u_{k-1} (host, 32 B each).  accumulate != 0 adds into dst instead: the
 * `msm.add_to_g_scalars(&compute_s(&u, neg_c))` of Guard::use_challenges (:36-41, msm.rs:104-113) without materialising s.
 * Fails for k == 0 like the reference's assert (:157).  Asynchronous. */
int h2_poly_compute_s(uint64_t dst, const void *u, uint32_t k, const void *init, int accumulate, int repr);
/* dst[i] = a * dst[i] + b * src[i] for i < n; src == 0: dst[i] = a * dst[i] (b ignored).  MSM::scale's g_scalars loop
 * (msm.rs:126-131), the g_scalars part of MSM::add_msm (msm.rs:52-54: a = 1, b = 1), and BatchVerifier's
 * `acc.scale(random); acc.add_msm(&msm)` (plonk/verifier/batch.rs:83-93) in one pass.  Asynchronous. */
int h2_poly_scale_add(uint64_t dst, const void *a, uint64_t src, const void *b, size_t n, int repr);

/* ---- key generation ------------------------------------------------------------------------------------------------ */
/* The permutation argument's sigma polynomials (plonk/permutation/keygen.rs:102-211) on resident polynomials:
 * dst[i][j] = delta^c * omega^r for (c, r) = mapping[2 (i n + j)], mapping[2 (i n + j) + 1], i < cols, j < n = 2^k.
 * mapping: cols * n pairs of uint32 (column, row) in host memory (pageable or pinned) -- the reference's
 * Assembly::mapping.  omega = domain.get_omega(), delta = F::DELTA, both in `repr`.  Fails when an entry is out of
 * range (the outputs are then unspecified), a handle is unknown / of another field / shorter than n, two dst handles are
 * equal, or k > 30; cols == 0 does nothing.  Synchronous. */
int h2_poly_permutation_sigma(const uint64_t *dst, size_t cols, uint32_t k, const uint32_t *mapping,
                              const void *omega, const void *delta, int repr);
/* The same sigma polynomials from the copy constraints themselves: the reference's Assembly (keygen.rs:24-100) runs on
 * the device (spanning forest of the copies, then the cycles by pointer jumping), with no mapping built or uploaded.
 * copies: m * 4 uint32 (left column, left row, right column, right row) in host memory, in synthesis order, columns as
 * indices into the permutation's column list.  Fails, with the index of the first bad copy and whether its column
 * (Error::ColumnNotInPermutation) or its row (Error::BoundsFailure) is out of range, and then writes nothing to dst.
 * Also fails on the checks of h2_poly_permutation_sigma, on cols * 2^k >= 2^32 and on m >= 2^32.  m == 0 gives the
 * identity sigma delta^c omega^r; cols == 0 does nothing.  Synchronous. */
int h2_poly_permutation_sigma_copies(const uint64_t *dst, size_t cols, uint32_t k, const uint32_t *copies, size_t m,
                                     const void *omega, const void *delta, int repr);

/* ---- the prover's product columns ------------------------------------------------------------------------------------ */
/* The permutation argument's product columns, permutation::Argument::commit (plonk/permutation/prover.rs:98-168), for
 * every set of every proof in one call.  The argument's `cols` columns are split into sets = ceil(cols / chunk_len) sets of
 * chunk_len (the last may be shorter); columns[p cols + c] is column c of proof p (any resident Lagrange column: advice,
 * fixed or instance, in the argument's column order), sigmas[c] its permutation polynomial.  z_out[p sets + a] receives
 * set a of proof p: the running product of
 *   prod_j (v_j[i] + beta delta^(c0 + j) omega^i + gamma) / (v_j[i] + beta sigma_j[i] + gamma)   (c0 = a chunk_len)
 * (a zero denominator counts as zero, ff::BatchInvert) starting at ONE for set 0 and at the previous set's row n - bf - 1
 * after it (last_z), with rows [n - bf, n) = blinding[(p sets + a) bf .. + bf) (the rng's order: per proof, per set).
 * omega = domain.get_omega(), delta = F::DELTA; scalars and blinding values in `repr`.
 * The inputs are only read, so shared polynomials (a shared proving key's sigma) work on every lane; z_out must be the
 * calling context's own, pairwise distinct and none of the inputs.  Every check runs before anything is launched, and a
 * failed check writes nothing: unknown handle, other field, fewer than n = 2^k elements, shared z_out, aliasing,
 * chunk_len == 0, blinding_factors + 1 >= n, k > 30, more than 65535 product columns.  proofs == 0 or cols == 0 does
 * nothing.  Asynchronous. */
int h2_poly_permutation_product(const uint64_t *z_out, size_t proofs, const uint64_t *columns, const uint64_t *sigmas, size_t cols,
                                uint32_t chunk_len, uint32_t k, const void *beta, const void *gamma, const void *omega, const void *delta,
                                const void *blinding, uint32_t blinding_factors, int repr);
/* The lookup argument's product columns, lookup::Permuted::commit_product (plonk/lookup/prover.rs:279-337), for `count`
 * lookups (of any number of proofs) in one call: z_out[b][0] = 1, z_out[b][i] = prod_(j < i) (a[j] + beta) (s[j] + gamma) /
 * ((beta + a'[j]) (gamma + s'[j])) for i < n - bf, rows [n - bf, n) = blinding[b bf .. + bf), where a = inputs[b],
 * s = tables[b] are the compressed columns and a' = permuted_inputs[b], s' = permuted_tables[b] the permuted ones (blinding
 * rows included).  Inputs, checks and asynchrony as h2_poly_permutation_product; count == 0 does nothing. */
int h2_poly_lookup_product(const uint64_t *z_out, size_t count, const uint64_t *inputs, const uint64_t *tables,
                           const uint64_t *permuted_inputs, const uint64_t *permuted_tables, uint32_t k, const void *beta,
                           const void *gamma, const void *blinding, uint32_t blinding_factors, int repr);

/* Reference sort of the MSM: by default every (point, window) reference is binned in ONE pass into fixed-capacity
 * per-bucket bins, with an automatic fallback to the exact histogram / scan / scatter sort when a bin overflows
 * (heavily repeated scalars).  exact_only != 0 forces the exact sort.  Same result; for A/B runs and tests. */
int h2_set_sort_mode(int exact_only);
/* GLV endomorphism split (k = k1 + k2 lambda, 129-bit halves; on by default) for MSMs without a
 * window table.  Same result; switchable for A/B measurements and tests. */
int h2_set_glv(int on);

/* Device-resident MSM: d_scalars (n x 32 B, `scalars_repr`), d_bases (n x 64 B, Montgomery),
 * d_out_xyz (96 B, Montgomery).  window_bits 0 = automatic.  Asynchronous on `stream`: the MSM runs after the caller's
 * earlier work on `stream` and after the calling context's earlier calls, and the context's later calls run after it.
 * Other lanes are unaffected. */
int h2_msm_dev(int curve, const void *d_scalars, int scalars_repr, const void *d_bases, size_t n,
               uint32_t window_bits, void *d_out_xyz, void *stream);

/* Sum of g Jacobian points (host, 96 B each): the combine step after the multi-GPU
 * all-gather of per-shard partial results (SURVEY.md section 8(e)). */
int h2_point_sum(int curve, const void *points_xyz, size_t g, int repr, void *out_xyz);
/* The same sum on device pointers (Montgomery in and out), enqueued on `stream`: the combine step directly behind an NCCL
 * all-gather, no host round trip. */
int h2_point_sum_dev(int curve, const void *d_points_xyz, size_t g, void *d_out_xyz, void *stream);

/* ---- single-process multi-GPU: SURVEY.md section 8(b) `h2_msm_multi_gpu`, section 8(e) --------------------------- */
/* best_multiexp (arithmetic.rs:143-180) is called from ONE process: after h2_init(primary), h2_multi_init(ngpu) binds
 * contexts to ngpu devices (the primary first, then the others in index order) and enables peer access.  h2_msm_multi_gpu
 * is h2_msm sharded over them: device g receives pairs [g n / G, (g + 1) n / G) (one worker thread per device, uploads in
 * parallel), runs the whole single-GPU pipeline, writes its 96-byte partial result into the primary device's memory over
 * NVLink, and the primary adds the G partial results.  Same group element as h2_msm for every ngpu. */
int h2_multi_init(int ngpu);
int h2_multi_count(void);
int h2_msm_multi_gpu(int curve, const void *scalars, const void *bases_xy, size_t n, int repr, void *out_xyz);
/* Bases resident per shard (the Params generators of a prover session; BASELINE configs[4]: "bases pre-resident"):
 * h2_msm_multi_registered then ships only the scalars. */
int h2_multi_bases_register(int curve, const void *bases_xy, size_t n, int repr, uint64_t *handle);
int h2_multi_bases_release(uint64_t handle);
int h2_msm_multi_registered(uint64_t handle, const void *scalars, size_t n, int repr, void *out_xyz);

/* ---- NTT: replaces best_fft for G = Scalar, arithmetic.rs:192-295 --------------------------- */
/* In-place radix-2 network on 2^log_n elements with the given omega (any field element,
 * not necessarily a root of unity -- benches/fft.rs:17). */
int h2_ntt(int field, void *a, const void *omega, uint32_t log_n, int repr);
/* EvaluationDomain::ifft (poly/domain.rs:375-383) == lagrange_to_coeff (:227-237):
 * best_fft with omega_inv, then a[i] *= divisor. */
int h2_intt_scaled(int field, void *a, const void *omega_inv, const void *divisor, uint32_t log_n, int repr);
/* EvaluationDomain::coeff_to_extended (poly/domain.rs:241-255): a has 2^k elements, out 2^ext_k.
 * zeta = F::ZETA (g_coset, :85). */
int h2_coeff_to_extended(int field, const void *a, uint32_t k, uint32_t ext_k, const void *zeta,
                         const void *ext_omega, void *out, int repr);
/* EvaluationDomain::extended_to_coeff (poly/domain.rs:303-325): a has 2^ext_k elements,
 * out receives the first out_len (= n * quotient_poly_degree) coefficients. */
int h2_extended_to_coeff(int field, const void *a, uint32_t ext_k, const void *ext_omega_inv,
                         const void *ext_divisor, const void *zeta, size_t out_len, void *out, int repr);

/* Device-resident NTT on Montgomery data; omega is a HOST pointer in `omega_repr`.
 * d_out may equal d_in.  mode: 0 = plain, see the host variants for the scaled forms.  Asynchronous on `stream`: the
 * transform runs after the caller's earlier work on `stream` and after the calling context's earlier calls, and the
 * context's later calls run after it.  Other lanes are unaffected. */
int h2_ntt_dev(int field, const void *d_in, void *d_out, const void *omega, int omega_repr, uint32_t log_n,
               void *stream);
/* Drops cached twiddle tables (the next call rebuilds them: "cold" timing). */
int h2_ntt_clear_cache(void);

/* ---- EC-FFT and batch normalisation: SURVEY.md section 8 rows a15 and (f)2 / (f)4 ------------------- */
/* best_fft at G = C::Curve (arithmetic.rs:192-295 through the FftGroup bound :17-27; call site
 * poly/commitment.rs:81-82): in-place butterfly network on 2^log_n Jacobian points (96 B x||y||z, z = 0 identity) with
 * scalar-field twiddles omega^i, then -- when `scale` is not NULL -- every output multiplied by the scalar `scale`
 * (`*g *= minv`, poly/commitment.rs:84-89).  omega / scale are elements of the curve's SCALAR field. */
int h2_ec_fft(int curve, void *points_xyz, const void *omega, uint32_t log_n, const void *scale, int repr);
/* group::Curve::batch_normalize (call sites plonk/prover.rs:99,311; poly/commitment.rs:65,95; vanishing/prover.rs:108):
 * n Jacobian points -> n affine points (64 B, identity = zeros), one inversion per 16 points. */
int h2_batch_normalize(int curve, const void *points_xyz, size_t n, int repr, void *out_xy);
/* The g -> g_lagrange derivation of Params::new (poly/commitment.rs:74-101) without leaving the device: affine g
 * (2^k x 64 B) -> EC-iFFT with omega_inv (= alpha_inv, :77-80) -> * minv (= 2^-k, :83-89) -> batch_normalize (:91-101)
 * -> affine g_lagrange.  (hash_to_curve, :46-58, lives in the un-vendored pasta_curves: the generators are the caller's.) */
int h2_params_lagrange(int curve, const void *g_xy, uint32_t k, const void *omega_inv, const void *minv, int repr, void *out_g_lagrange_xy);
/* C::CurveExt::hash_to_curve(domain_prefix)(message) (call sites poly/commitment.rs:52,102; benches/hashtocurve.rs:15,18;
 * the implementation is pasta_curves 0.5.1 src/hashtocurve.rs, un-vendored): the RFC 9380 suite
 * "<curve>_XMD:BLAKE2b_SSWU_RO_" -- expand_message_xmd over BLAKE2b-512, simplified SWU onto the 3-isogenous curve
 * y^2 = x^3 + A x + 1265 (Z = -13), sum of the two images, 3-isogeny back.  n messages of msg_len bytes each (stride
 * msg_len) -> n affine points (64 B).  Pinned on the reference's golden commitments (tests/plonk_api.rs:958-982). */
int h2_hash_to_curve(int curve, const char *domain_prefix, const void *messages, size_t msg_len, size_t n, int repr, void *out_xy);
/* Params::new(k) whole (poly/commitment.rs:38-114): g[i] = H(0 || i as u32 LE) (:46-58), w = H([1]), u = H([2]) (:102-105)
 * with H = hash_to_curve("Halo2-Parameters"), and g_lagrange = batch_normalize(2^-k * EC-iFFT(g)) (:74-101), all on the
 * device.  Outputs: g and g_lagrange 2^k x 64 B, w and u 64 B each. */
int h2_params_new(int curve, uint32_t k, int repr, void *out_g_xy, void *out_g_lagrange_xy, void *out_w_xy, void *out_u_xy);

/* ---- point encoding: SURVEY.md section 8(f) row 4 (the wire format either side of the path) ----------------------- */
/* C::to_bytes (book/src/background/curves.md:203-225): n affine points (64 B) -> n x 32 bytes, x little-endian with the LSB
 * of y in the top bit of the last byte, identity = zeros.  What Params::write (poly/commitment.rs:168-181) and the
 * transcript (transcript.rs: write_point) emit for every point. */
int h2_points_compress(int curve, const void *points_xy, size_t n, int repr, void *out_bytes);
/* C::from_bytes (curves.md:227-240): y = sqrt(x^3 + 5) with the encoded sign (Tonelli-Shanks on the device).  Fails -- like
 * C::read's io::Error in Params::read, poly/commitment.rs:183-205 -- when an encoding is invalid (x not canonical, x = 0 with
 * the sign bit set, x^3 + 5 not a square); h2_last_error() names the first bad index. */
int h2_points_decompress(int curve, const void *bytes, size_t n, int repr, void *out_xy);

/* ---- utilities for synthetic workloads and the tests ---------------------------------------- */
/* d_out[i] = [s_i] * (-1, 2) for pseudo-random 64-bit s_i derived from seed (distinct points),
 * affine Montgomery coordinates; i in [first, first + n). */
int h2_dev_gen_points(int curve, uint64_t seed, uint64_t first, size_t n, void *d_out, void *stream);
/* In-place canonical <-> Montgomery conversion of n field elements on the device. */
int h2_dev_convert(int field, void *d_a, size_t n, int to_montgomery, void *stream);
/* Test hook: bit 0 = the most recent MSM split some bucket over several work items, bit 1 = it used the exact
 * (two-pass) sort.  Synchronises the device. */
int h2_test_last_msm_flags(uint32_t *out);
/* Test hook: what the most recent MSM pass over at least one term ran, recorded on the host (graph replays included):
 *   out[0] mode: 0 one-shot (no table), 1 window table, 2 digit-multiples table (direct sum)
 *   out[1] window bits c   out[2] windows W   out[3] scalar vectors in the pass (sets)
 *   out[4] accumulation: 0 cooperating lanes per work item, 1 a thread per work item (msm_accum0_kernel and the partial-merge
 *          levels), 2 the direct sum of mode 2
 *   out[5] natural (work items = the buckets in index order)   out[6] fast (fixed-base pass without the fallback kernels)
 *   out[7] 1 if this pass re-ran, in full, a fast pass whose device flags came back set
 * Fails if no MSM has run. */
int h2_test_last_msm_plan(uint32_t out[8]);
/* Test hook: h2_msm uploads the bases of inputs with >= 2^log2_n points in chunks that are sorted and accumulated
 * separately while the next chunk is on the PCIe link (default 19). */
int h2_test_set_chunk_threshold(uint32_t log2_n);
/* Tuning hook: the points at which a k-chunk upload (k = 2, 3, 4) is cut, in sixteenths of n: chunks GROW so that the upload
 * of chunk j + 1 hides behind the accumulation of chunk j (defaults 4 | 2, 8 | 1, 4, 10). */
int h2_test_set_chunk_cuts(uint32_t k, uint32_t c1, uint32_t c2, uint32_t c3);
/* Transfers from / to PAGEABLE caller memory (a Rust Vec) go through a pinned staging ring filled by a few host threads,
 * so that the link runs near its pinned rate and uploads still overlap compute; pinned / registered memory is used in
 * place.  0 switches the ring off (plain cudaMemcpyAsync): bench.py times both. */
int h2_test_set_staging(int on);
/* Staging-copy tuning: `threads` worker threads share every ring-slot copy with the calling thread (-1 keeps the current
 * value; default 15 on hosts with >= 64 hardware threads, else 7 / 3; env H2_COPY_THREADS overrides); nt_stores: 1 = AVX2
 * non-temporal stores into the pinned slot (default), 0 = memcpy, -1 keeps. */
int h2_test_set_copy_threads(int threads, int nt_stores);
/* 1: NTT passes run as a persistent kernel whose tile traffic is on the bulk-copy (TMA) engine (cp.async.bulk + mbarrier,
 * double buffered) wherever the pass geometry allows; 0 (default -- measured faster on H100, ctx.cuh): the classic
 * load / compute / store kernel.  bench.py times both. */
int h2_test_set_ntt_tma(int on);
/* Fixed-base MSMs over resident window tables first run WITHOUT their fallback kernels (the exact two-pass sort and the merge of
 * split buckets: 10 of ~27 graph nodes that do nothing on ordinary scalars); the two device flags come back with the result
 * and a set flag -- a constant or 0/1 column, for instance -- re-runs the full pass.  1 (default) / 0 = always the full pass.
 * Tuning values: 2 = fast passes never take their buckets in index order; v >= 3 = they do up to 2^v buckets (default 14). */
int h2_test_set_fast_fixed(int on);
/* Opt-in: h2_poly_eval / h2_poly_kate_division on polynomials of up to 2^16 coefficients in ONE launch, one CTA per polynomial
 * (1); 0 (default) = the tree of 32-coefficient levels, which fills the machine (ctx.cuh). */
int h2_test_set_poly_cta(int on);
/* Test hook: fixed-base MSMs over resident bases replay a captured CUDA graph from their third call with the same
 * parameters on (default); 0 issues every launch individually. */
int h2_test_set_graphs(int on);
/* EC-FFT butterfly form: 1 = quads of lanes, 0 = one thread each, -1 = chosen by size (the default). */
int h2_test_set_ecfft_quad(int on);
/* Opt-in: large one-shot MSMs add their buckets' points pairwise in AFFINE coordinates first -- `rounds` halving rounds (0 = off,
 * the default; at most 3), one shared inversion per `pairs_per_thread` additions (0 keeps the value) -- and finish with the
 * XYZZ chain.  6 multiplies per addition instead of 10, but measured slower on H100 (ctx.cuh).  Tuning: bits 8.. of
 * `rounds` select the kernel variant + 1 (gather chunk of 4 / 2 pairs at 4 / 5 CTAs per SM); bit 16 of `pairs_per_thread` keeps that
 * many pairs per thread in every round instead of keeping the thread count. */
int h2_test_set_batched_affine(uint32_t rounds, uint32_t pairs_per_thread);
/* Lanes per work item in the accumulation of small MSMs: 12 / 14 = 2 / 4 independent lanes (12 is the default), 0 = one cooperating
 * pair of lanes, 1, 2 or 4 = quads (measurements in ctx.cuh).
 * Tuning: bits 8.. of `ways`, when non-zero, set log2 of the reference count up to which lanes cooperate (default 20; fixed-base
 * passes use twice that). */
int h2_test_set_accum_ways(uint32_t ways);
/* Self-test kernels used by tests/: out[i] = a[i] (op) b[i] on the device, canonical bytes,
 * host buffers.  op: 0 add, 1 sub, 2 mul, 3 inverse(a) by the Fermat ladder,
 * 4 square(a), 5 inverse(a) by division steps (fe_inv_gcd, what the kernels use). */
int h2_test_field_op(int field, int op, const void *a, const void *b, size_t n, void *out);
/* Self-test of the device group law; canonical affine points in and out, identity = (0, 0), host buffers.
 *   op 0  a[i] + b[i] by the mixed and the full addition (the poison point (1, 0) if they disagree)
 *   op 1  2 a[i]            op 2  k[i] * a[i], b = 32-byte scalars padded to 64 B
 * Ops 3 .. 13 run one form each on XYZZ operands rescaled by a per-element factor l (X = l^2 x, Y = l^3 y, ZZ = l^2,
 * ZZZ = l^3; l = 1 for i % 4 == 0), the two operands of a full addition with independent factors:
 *   op 3  xyzz_add            a[i] + b[i]     op 4  xyzz_add_mixed   a[i] + b[i] (b affine)
 *   op 5  xyzz_double         2 a[i]          op 6  xyzz_shift       2^k a[i], k = the low 32 bits of b[i].x
 * Ops 7 .. 13 are the lane-cooperative forms, 4 lanes per element (op 9: 2); the result is the poison point if the lanes
 * of an element end with different values:
 *   op 7  xyzz_add_quad       a[i] + b[i]     op 8  xyzz_add_mixed_quad   a[i] + b[i] (b affine)
 *   op 9  xyzz_add_mixed_pair a[i] + b[i]     op 10 xyzz_shift_quad       2^k a[i], k as in op 6
 *   op 11 / 12  xyzz_addsub_q<P, true>   a[i] + b[i] / a[i] - b[i]        op 13 xyzz_double_q   2 a[i]
 * Any other op fails. */
int h2_test_curve_op(int curve, int op, const void *a_xy, const void *b_xy, size_t n, void *out_xy);
/* Times `iters` dependent field multiplications per thread over `threads` threads; returns
 * elapsed milliseconds in *ms (microbenchmark for the roofline discussion in DESIGN.md). */
int h2_bench_field_mul(int field, uint32_t threads_per_block, uint32_t blocks, uint32_t iters, float *ms);
/* Single-warp latency of the serial building blocks: mode 0 dependent multiply chain, 1 two
 * independent chains, 2 four chains, 3 xyzz double, 4 xyzz add, 5 xyzz mixed add. */
int h2_bench_latency(int mode, uint32_t iters, float *ms);
/* Number of kernels launched by the engine since h2_init (bench.py's gpu_launches). */
uint64_t h2_launch_count(void);
/* Per-kernel device timing for the roofline report: while enabled, CUDA-event pairs bracket the
 * dominant kernels on their launch stream.  kind 0 = MSM bucket-accumulate kernel, 1 = NTT pass
 * kernel.  h2_profile_enable(0/1) also clears the recorded spans. */
int h2_profile_enable(int on);
int h2_profile_read(int kind, float *total_ms, uint32_t *launches);

#ifdef __cplusplus
}
#endif
#endif /* HALO2_B200_H */
