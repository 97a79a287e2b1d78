/*
 * CPU oracle, C restatement (TEST INFRASTRUCTURE + the timed "reference algorithm" CPU
 * baseline).  NOT part of the product: only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load this library.
 *
 * Restates, for the Pasta fields/curves (file:line relative to
 * /root/reference/halo2_proofs/src):
 *   best_multiexp      arithmetic.rs:143-180 with Bucket/Buckets :29-112 -- same window size
 *                      c (:146-152), 256/c+1 windows (:154), unsigned digits from the canonical
 *                      LE repr (get_at :95-111), None->Affine->Projective buckets (:37-46),
 *                      summation by parts (:86-92), one task per window when n > threads
 *                      (:157-167) else serial Horner (:168-179).
 *   best_fft           arithmetic.rs:192-255 + recursive_butterfly_arithmetic :258-295:
 *                      serial bit reversal (:207-212), serial twiddle scan (:215-221),
 *                      iterative stages when log_n <= log2(threads) else join-recursion.
 *   parallelize        arithmetic.rs:345-362 (chunk = n/threads; if chunk < threads one chunk).
 *   ifft / distribute_powers_zeta / coeff_to_extended / extended_to_coeff
 *                      poly/domain.rs:375-383, :357-373, :241-255, :303-325.
 *   best_fft (G = curve point), batch_normalize, g -> g_lagrange
 *                      arithmetic.rs:192-295 at G = C::Curve; poly/commitment.rs:74-101 (Params::new from the generators on).
 *   permute_expression_pair  plonk/lookup/prover.rs:563-647 (sort + ordered map restated as sorted table + taken marks; serial).
 *   product columns    plonk/permutation/prover.rs:81-168, plonk/lookup/prover.rs:279-321, with ff::BatchInvert; serial.
 *   divide_by_vanishing_poly  poly/domain.rs:329-348; serial.
 *   eval_polynomial, kate_division, Evaluator::evaluate (postfix form): see each section (hash_to_curve is restated in pasta.py only).
 *   IPA round loop     poly/commitment/prover.rs:100-142 with parallel_generator_collapse :154-166 and
 *                      compute_inner_product arithmetic.rs:308-319; the transcript is factored out (challenges and
 *                      randomness are inputs).
 *
 * The limb arithmetic itself lives in the un-vendored crate pasta_curves 0.5.1
 * (Cargo.lock:1303-1306); it is restated from the definition (4x64 Montgomery, R = 2^256).
 * The reference is Rust-only and cannot be compiled in this image, so there is no
 * oracle/_ref; bench.py reports this library as cpu_baseline.kind = "port".
 *
 * PARITY PINNING: PINNED on reference-held vectors -- this library's EC-FFT (orc_params_lagrange) fed with the
 * hash_to_curve generators and its threaded best_multiexp reproduce all 19 golden commitments of the plonk_api
 * verifying key (tests/plonk_api.rs:958-982; tests/test_oracle_golden.py::test_golden_commitments_c_oracle); the field
 * layer is pinned by the halo2_poseidon known-answer vectors.  See the oracle/pasta.py header for the full status.
 *
 * ABI: every element is canonical 32-byte little-endian; affine point = x||y (64 B),
 * identity = 64 zero bytes.  field: 0 = Fp, 1 = Fq.  curve: 0 = Pallas (coords Fp, scalars
 * Fq), 1 = Vesta (coords Fq, scalars Fp).
 */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef unsigned __int128 u128;
typedef struct { uint64_t l[4]; } fe;           /* Montgomery form */
typedef struct { fe x, y; int inf; } aff;       /* affine, inf=1 identity */
typedef struct { fe x, y, z; } jac;             /* Jacobian, z==0 identity */

typedef struct {
    uint64_t m[4];   /* modulus */
    uint64_t inv;    /* -m^-1 mod 2^64 */
    fe r;            /* R mod m (Montgomery one) */
    fe r2;           /* R^2 mod m */
} field_t;

static field_t FLD[2];
static int g_init = 0;

static const uint64_t MOD_P[4] = {0x992d30ed00000001ULL, 0x224698fc094cf91bULL, 0x0ULL, 0x4000000000000000ULL};
static const uint64_t MOD_Q[4] = {0x8c46eb2100000001ULL, 0x224698fc0994a8ddULL, 0x0ULL, 0x4000000000000000ULL};

/* ---------------------------------------------------------------- limb helpers */
static inline int ge4(const uint64_t *a, const uint64_t *b) {
    for (int i = 3; i >= 0; i--) { if (a[i] > b[i]) return 1; if (a[i] < b[i]) return 0; }
    return 1;
}
static inline uint64_t sub4(uint64_t *r, const uint64_t *a, const uint64_t *b) {
    uint64_t borrow = 0;
    for (int i = 0; i < 4; i++) {
        u128 d = (u128)a[i] - b[i] - borrow;
        r[i] = (uint64_t)d; borrow = (uint64_t)(d >> 64) & 1;
    }
    return borrow;
}
static inline uint64_t add4(uint64_t *r, const uint64_t *a, const uint64_t *b) {
    uint64_t carry = 0;
    for (int i = 0; i < 4; i++) {
        u128 s = (u128)a[i] + b[i] + carry;
        r[i] = (uint64_t)s; carry = (uint64_t)(s >> 64);
    }
    return carry;
}

static inline void fe_add(const field_t *F, fe *r, const fe *a, const fe *b) {
    uint64_t t[4]; add4(t, a->l, b->l);            /* < 2m < 2^256: no carry */
    if (ge4(t, F->m)) sub4(t, t, F->m);
    memcpy(r->l, t, 32);
}
static inline void fe_sub(const field_t *F, fe *r, const fe *a, const fe *b) {
    uint64_t t[4];
    if (sub4(t, a->l, b->l)) add4(t, t, F->m);
    memcpy(r->l, t, 32);
}
static inline void fe_neg(const field_t *F, fe *r, const fe *a) {
    fe z = {{0, 0, 0, 0}}; fe_sub(F, r, &z, a);
}
static inline int fe_is_zero(const fe *a) { return (a->l[0] | a->l[1] | a->l[2] | a->l[3]) == 0; }
static inline int fe_eq(const fe *a, const fe *b) { return memcmp(a->l, b->l, 32) == 0; }

/* CIOS Montgomery multiplication, 4 x 64-bit limbs */
static inline void fe_mul(const field_t *F, fe *r, const fe *a, const fe *b) {
    uint64_t t[6] = {0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 4; i++) {
        uint64_t c = 0;
        for (int j = 0; j < 4; j++) {
            u128 s = (u128)a->l[j] * b->l[i] + t[j] + c;
            t[j] = (uint64_t)s; c = (uint64_t)(s >> 64);
        }
        u128 s = (u128)t[4] + c; t[4] = (uint64_t)s; t[5] = (uint64_t)(s >> 64);
        uint64_t q = t[0] * F->inv;
        s = (u128)q * F->m[0] + t[0]; c = (uint64_t)(s >> 64);
        for (int j = 1; j < 4; j++) {
            s = (u128)q * F->m[j] + t[j] + c;
            t[j - 1] = (uint64_t)s; c = (uint64_t)(s >> 64);
        }
        s = (u128)t[4] + c; t[3] = (uint64_t)s; t[4] = t[5] + (uint64_t)(s >> 64);
    }
    if (t[4] || ge4(t, F->m)) sub4(t, t, F->m);
    memcpy(r->l, t, 32);
}
static inline void fe_sqr(const field_t *F, fe *r, const fe *a) { fe_mul(F, r, a, a); }

static void fe_from_bytes(const field_t *F, fe *r, const uint8_t *b) {
    fe t; memcpy(t.l, b, 32);                      /* little-endian host assumed */
    fe_mul(F, r, &t, &F->r2);
}
static void fe_to_bytes(const field_t *F, uint8_t *b, const fe *a) {
    fe one = {{1, 0, 0, 0}}, t; fe_mul(F, &t, a, &one);
    memcpy(b, t.l, 32);
}
static void fe_pow(const field_t *F, fe *r, const fe *a, const uint64_t e[4]) {
    fe acc = F->r, base = *a;
    for (int i = 0; i < 256; i++) {
        if ((e[i >> 6] >> (i & 63)) & 1) fe_mul(F, &acc, &acc, &base);
        fe_sqr(F, &base, &base);
    }
    *r = acc;
}
static void fe_inv(const field_t *F, fe *r, const fe *a) {
    uint64_t e[4] = {F->m[0] - 2, F->m[1], F->m[2], F->m[3]};
    fe_pow(F, r, a, e);
}

static void field_setup(field_t *F, const uint64_t m[4]) {
    memcpy(F->m, m, 32);
    uint64_t x = 1;                                /* Newton: x = m^-1 mod 2^64 */
    for (int i = 0; i < 6; i++) x *= 2 - m[0] * x;
    F->inv = (uint64_t)0 - x;
    /* R mod m by 256 modular doublings of 1, R^2 by 512 */
    uint64_t t[4] = {1, 0, 0, 0};
    for (int i = 0; i < 512; i++) {
        uint64_t c = add4(t, t, t);
        if (c || ge4(t, m)) sub4(t, t, m);
        if (i == 255) memcpy(F->r.l, t, 32);
    }
    memcpy(F->r2.l, t, 32);
}
static void ensure_init(void) {
    if (g_init) return;
    field_setup(&FLD[0], MOD_P);
    field_setup(&FLD[1], MOD_Q);
    g_init = 1;
}
static inline const field_t *base_field(int curve) { return &FLD[curve]; }       /* pallas->fp */
static inline const field_t *scalar_field(int curve) { return &FLD[1 - curve]; } /* pallas->fq */

/* ---------------------------------------------------------------- curve: y^2 = x^3 + 5 */
static inline void jac_identity(const field_t *F, jac *r) {
    memset(r, 0, sizeof *r); r->y = F->r;
}
static inline int jac_is_id(const jac *a) { return fe_is_zero(&a->z); }

static void jac_double(const field_t *F, jac *r, const jac *p) {
    if (jac_is_id(p)) { *r = *p; return; }
    fe A, B, C, D, E, Ff, t, X3, Y3, Z3;
    fe_sqr(F, &A, &p->x); fe_sqr(F, &B, &p->y); fe_sqr(F, &C, &B);
    fe_add(F, &t, &p->x, &B); fe_sqr(F, &t, &t); fe_sub(F, &t, &t, &A); fe_sub(F, &t, &t, &C);
    fe_add(F, &D, &t, &t);
    fe_add(F, &E, &A, &A); fe_add(F, &E, &E, &A);
    fe_sqr(F, &Ff, &E);
    fe_sub(F, &X3, &Ff, &D); fe_sub(F, &X3, &X3, &D);
    fe_sub(F, &t, &D, &X3); fe_mul(F, &Y3, &E, &t);
    fe_add(F, &C, &C, &C); fe_add(F, &C, &C, &C); fe_add(F, &C, &C, &C);
    fe_sub(F, &Y3, &Y3, &C);
    fe_mul(F, &Z3, &p->y, &p->z); fe_add(F, &Z3, &Z3, &Z3);
    r->x = X3; r->y = Y3; r->z = Z3;
}

static void jac_add(const field_t *F, jac *r, const jac *a, const jac *b) {
    if (jac_is_id(a)) { *r = *b; return; }
    if (jac_is_id(b)) { *r = *a; return; }
    fe z1z1, z2z2, u1, u2, s1, s2, h, rr, hh, hhh, v, t, X3, Y3, Z3;
    fe_sqr(F, &z1z1, &a->z); fe_sqr(F, &z2z2, &b->z);
    fe_mul(F, &u1, &a->x, &z2z2); fe_mul(F, &u2, &b->x, &z1z1);
    fe_mul(F, &s1, &a->y, &b->z); fe_mul(F, &s1, &s1, &z2z2);
    fe_mul(F, &s2, &b->y, &a->z); fe_mul(F, &s2, &s2, &z1z1);
    if (fe_eq(&u1, &u2)) {
        if (fe_eq(&s1, &s2)) { jac_double(F, r, a); return; }
        jac_identity(F, r); return;
    }
    fe_sub(F, &h, &u2, &u1); fe_sub(F, &rr, &s2, &s1);
    fe_sqr(F, &hh, &h); fe_mul(F, &hhh, &h, &hh); fe_mul(F, &v, &u1, &hh);
    fe_sqr(F, &X3, &rr); fe_sub(F, &X3, &X3, &hhh); fe_sub(F, &X3, &X3, &v); fe_sub(F, &X3, &X3, &v);
    fe_sub(F, &t, &v, &X3); fe_mul(F, &Y3, &rr, &t); fe_mul(F, &t, &s1, &hhh); fe_sub(F, &Y3, &Y3, &t);
    fe_mul(F, &Z3, &a->z, &b->z); fe_mul(F, &Z3, &Z3, &h);
    r->x = X3; r->y = Y3; r->z = Z3;
}

static void jac_add_mixed(const field_t *F, jac *r, const jac *a, const aff *b) {
    if (b->inf) { *r = *a; return; }
    if (jac_is_id(a)) { r->x = b->x; r->y = b->y; r->z = F->r; return; }
    fe z1z1, u2, s2, h, rr, hh, hhh, v, t, X3, Y3, Z3;
    fe_sqr(F, &z1z1, &a->z);
    fe_mul(F, &u2, &b->x, &z1z1);
    fe_mul(F, &s2, &b->y, &a->z); fe_mul(F, &s2, &s2, &z1z1);
    if (fe_eq(&a->x, &u2)) {
        if (fe_eq(&a->y, &s2)) { jac_double(F, r, a); return; }
        jac_identity(F, r); return;
    }
    fe_sub(F, &h, &u2, &a->x); fe_sub(F, &rr, &s2, &a->y);
    fe_sqr(F, &hh, &h); fe_mul(F, &hhh, &h, &hh); fe_mul(F, &v, &a->x, &hh);
    fe_sqr(F, &X3, &rr); fe_sub(F, &X3, &X3, &hhh); fe_sub(F, &X3, &X3, &v); fe_sub(F, &X3, &X3, &v);
    fe_sub(F, &t, &v, &X3); fe_mul(F, &Y3, &rr, &t); fe_mul(F, &t, &a->y, &hhh); fe_sub(F, &Y3, &Y3, &t);
    fe_mul(F, &Z3, &a->z, &h);
    r->x = X3; r->y = Y3; r->z = Z3;
}

static void jac_to_aff(const field_t *F, aff *r, const jac *a) {
    if (jac_is_id(a)) { memset(r, 0, sizeof *r); r->inf = 1; return; }
    fe zi, zi2;
    fe_inv(F, &zi, &a->z); fe_sqr(F, &zi2, &zi);
    fe_mul(F, &r->x, &a->x, &zi2); fe_mul(F, &zi2, &zi2, &zi); fe_mul(F, &r->y, &a->y, &zi2);
    r->inf = 0;
}
static void aff_from_bytes(const field_t *F, aff *r, const uint8_t *b) {
    int allz = 1;
    for (int i = 0; i < 64; i++) if (b[i]) { allz = 0; break; }
    if (allz) { memset(r, 0, sizeof *r); r->inf = 1; return; }
    fe_from_bytes(F, &r->x, b); fe_from_bytes(F, &r->y, b + 32); r->inf = 0;
}
static void aff_to_bytes(const field_t *F, uint8_t *b, const aff *a) {
    if (a->inf) { memset(b, 0, 64); return; }
    fe_to_bytes(F, b, &a->x); fe_to_bytes(F, b + 32, &a->y);
}
static void scalar_mul_bytes(const field_t *F, jac *r, const uint8_t k[32], const aff *base) {
    jac acc; jac_identity(F, &acc);
    for (int i = 255; i >= 0; i--) {
        jac_double(F, &acc, &acc);
        if ((k[i >> 3] >> (i & 7)) & 1) jac_add_mixed(F, &acc, &acc, base);
    }
    *r = acc;
}

/* ---------------------------------------------------------------- best_multiexp */
/* Bucket enum, arithmetic.rs:29-58 */
typedef struct { int tag; aff a; jac p; } bucket_t;   /* 0 None, 1 Affine, 2 Projective */

static inline void bucket_add_assign(const field_t *F, bucket_t *b, const aff *other) {
    if (b->tag == 0) { b->a = *other; b->tag = 1; }
    else if (b->tag == 1) {                      /* a + *other -> projective (arithmetic.rs:41) */
        jac t;
        if (b->a.inf) jac_identity(F, &t); else { t.x = b->a.x; t.y = b->a.y; t.z = F->r; }
        jac_add_mixed(F, &b->p, &t, other); b->tag = 2;
    } else jac_add_mixed(F, &b->p, &b->p, other);
}
static inline void bucket_add(const field_t *F, const bucket_t *b, jac *other) {
    if (b->tag == 1) jac_add_mixed(F, other, other, &b->a);
    else if (b->tag == 2) jac_add(F, other, other, &b->p);
}
/* get_at, arithmetic.rs:95-111 */
static inline size_t get_at(size_t segment, size_t c, const uint8_t *bytes) {
    size_t skip_bits = segment * c, skip_bytes = skip_bits / 8;
    if (skip_bytes >= 32) return 0;
    uint8_t v[8] = {0};
    for (size_t i = 0; i < 8 && skip_bytes + i < 32; i++) v[i] = bytes[skip_bytes + i];
    uint64_t tmp; memcpy(&tmp, v, 8);
    tmp >>= skip_bits - skip_bytes * 8;
    return (size_t)(tmp % ((uint64_t)1 << c));
}
/* Buckets::sum, arithmetic.rs:74-93 */
static void buckets_sum(const field_t *F, size_t c, const uint8_t *reprs, const aff *bases, size_t n,
                        size_t win, bucket_t *buckets, jac *out) {
    size_t nb = ((size_t)1 << c) - 1;
    for (size_t i = 0; i < nb; i++) buckets[i].tag = 0;
    for (size_t i = 0; i < n; i++) {
        size_t seg = get_at(win, c, reprs + 32 * i);
        if (seg) bucket_add_assign(F, &buckets[seg - 1], &bases[i]);
    }
    jac acc, sum; jac_identity(F, &acc); jac_identity(F, &sum);
    for (size_t i = nb; i-- > 0;) {
        bucket_add(F, &buckets[i], &sum);
        jac_add(F, &acc, &acc, &sum);
    }
    *out = acc;
}

typedef struct {
    const field_t *F; size_t c, n, windows; const uint8_t *reprs; const aff *bases;
    jac *results; volatile long next; pthread_mutex_t mu;
} msm_job;

static void *msm_worker(void *arg) {
    msm_job *J = (msm_job *)arg;
    bucket_t *buckets = (bucket_t *)malloc(sizeof(bucket_t) * (((size_t)1 << J->c) - 1));
    for (;;) {
        pthread_mutex_lock(&J->mu);
        long w = J->next; if (w >= 0) J->next = w - 1;    /* .rev(): top window first */
        pthread_mutex_unlock(&J->mu);
        if (w < 0) break;
        jac acc;
        buckets_sum(J->F, J->c, J->reprs, J->bases, J->n, (size_t)w, buckets, &acc);
        for (size_t d = 0; d < J->c * (size_t)w; d++) jac_double(J->F, &acc, &acc);   /* :163 */
        J->results[w] = acc;
    }
    free(buckets);
    return NULL;
}

static size_t window_bits(size_t n) {               /* arithmetic.rs:146-152 */
    if (n < 4) return 1;
    if (n < 32) return 3;
    return (size_t)ceil(log((double)(uint32_t)n));
}

/* scalars: n x 32 B canonical; bases: n x 64 B canonical affine; out: 64 B affine.
 * threads plays the role of rayon's current_num_threads(). */
static void msm_core(const field_t *F, const uint8_t *scalars, const aff *pts, size_t n, int threads, jac *out);
int orc_best_multiexp(int curve, const uint8_t *scalars, const uint8_t *bases, size_t n, int threads,
                      uint8_t *out_xy) {
    ensure_init();
    if (threads < 1) threads = 1;
    const field_t *F = base_field(curve);
    aff *pts = (aff *)malloc(sizeof(aff) * (n ? n : 1));
    for (size_t i = 0; i < n; i++) aff_from_bytes(F, &pts[i], bases + 64 * i);
    jac total;
    msm_core(F, scalars, pts, n, threads, &total);
    aff r; jac_to_aff(F, &r, &total); aff_to_bytes(F, out_xy, &r);
    free(pts);
    return 0;
}
/* best_multiexp proper, arithmetic.rs:143-180, on decoded bases */
static void msm_core(const field_t *F, const uint8_t *scalars, const aff *pts, size_t n, int threads, jac *out) {
    size_t c = window_bits(n), windows = 256 / c + 1;
    jac total; jac_identity(F, &total);
    if (n > (size_t)threads) {
        msm_job J; J.F = F; J.c = c; J.n = n; J.windows = windows; J.reprs = scalars; J.bases = pts;
        J.results = (jac *)malloc(sizeof(jac) * windows); J.next = (long)windows - 1;
        pthread_mutex_init(&J.mu, NULL);
        int nt = threads < (int)windows ? threads : (int)windows;
        pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * nt);
        for (int t = 1; t < nt; t++) pthread_create(&th[t], NULL, msm_worker, &J);
        msm_worker(&J);
        for (int t = 1; t < nt; t++) pthread_join(th[t], NULL);
        for (size_t w = 0; w < windows; w++) jac_add(F, &total, &total, &J.results[w]);   /* :166 */
        free(th); free(J.results); pthread_mutex_destroy(&J.mu);
    } else {
        bucket_t *buckets = (bucket_t *)malloc(sizeof(bucket_t) * (((size_t)1 << c) - 1));
        for (size_t w = windows; w-- > 0;) {          /* :168-179 */
            for (size_t d = 0; d < c; d++) jac_double(F, &total, &total);
            jac acc; buckets_sum(F, c, scalars, pts, n, w, buckets, &acc);
            jac_add(F, &total, &total, &acc);
        }
        free(buckets);
    }
    *out = total;
}

/* naive sum_i k_i * P_i, the other side of test_multiexp (arithmetic.rs:440-458) */
int orc_naive_msm(int curve, const uint8_t *scalars, const uint8_t *bases, size_t n, uint8_t *out_xy) {
    ensure_init();
    const field_t *F = base_field(curve);
    jac total; jac_identity(F, &total);
    for (size_t i = 0; i < n; i++) {
        aff b; aff_from_bytes(F, &b, bases + 64 * i);
        jac t; scalar_mul_bytes(F, &t, scalars + 32 * i, &b);
        jac_add(F, &total, &total, &t);
    }
    aff r; jac_to_aff(F, &r, &total); aff_to_bytes(F, out_xy, &r);
    return 0;
}

/* ---------------------------------------------------------------- best_fft */
static int log2_floor(unsigned v) { int r = -1; while (v) { v >>= 1; r++; } return r; }  /* :364-374 */

typedef struct { const field_t *F; fe *a; size_t n, tc; const fe *tw; int depth; } fft_task;

static void butterflies(const field_t *F, fe *left, fe *right, size_t half, size_t tc, const fe *tw) {
    fe t = right[0];
    right[0] = left[0];
    fe_add(F, &left[0], &left[0], &t); fe_sub(F, &right[0], &right[0], &t);
    for (size_t i = 1; i < half; i++) {
        fe_mul(F, &t, &right[i], &tw[i * tc]);
        right[i] = left[i];
        fe_add(F, &left[i], &left[i], &t); fe_sub(F, &right[i], &right[i], &t);
    }
}
static void *fft_rec(void *arg) {                     /* arithmetic.rs:258-295 */
    fft_task *T = (fft_task *)arg;
    if (T->n == 2) {
        fe t = T->a[1]; T->a[1] = T->a[0];
        fe_add(T->F, &T->a[0], &T->a[0], &t); fe_sub(T->F, &T->a[1], &T->a[1], &t);
        return NULL;
    }
    size_t h = T->n / 2;
    fft_task L = {T->F, T->a, h, T->tc * 2, T->tw, T->depth - 1};
    fft_task R = {T->F, T->a + h, h, T->tc * 2, T->tw, T->depth - 1};
    if (T->depth > 0) {                               /* multicore::join */
        pthread_t th; pthread_create(&th, NULL, fft_rec, &L);
        fft_rec(&R); pthread_join(th, NULL);
    } else { fft_rec(&L); fft_rec(&R); }
    butterflies(T->F, T->a, T->a + h, h, T->tc, T->tw);
    return NULL;
}
static size_t bitrev(size_t n, unsigned l) { size_t r = 0; for (unsigned i = 0; i < l; i++) { r = (r << 1) | (n & 1); n >>= 1; } return r; }

static void fft_mont(const field_t *F, fe *a, const fe *omega, uint32_t log_n, int threads) {
    size_t n = (size_t)1 << log_n;
    int log_threads = log2_floor((unsigned)threads);
    for (size_t k = 0; k < n; k++) {
        size_t rk = bitrev(k, log_n);
        if (k < rk) { fe t = a[k]; a[k] = a[rk]; a[rk] = t; }
    }
    size_t nt = n / 2 ? n / 2 : 1;
    fe *tw = (fe *)malloc(sizeof(fe) * nt);
    fe w = F->r;
    for (size_t i = 0; i < n / 2; i++) { tw[i] = w; fe_mul(F, &w, &w, omega); }
    if ((int)log_n <= log_threads) {
        size_t chunk = 2, tc = n / 2;
        for (uint32_t s = 0; s < log_n; s++) {
            for (size_t base = 0; base < n; base += chunk)
                butterflies(F, a + base, a + base + chunk / 2, chunk / 2, tc, tw);
            chunk *= 2; tc /= 2;
        }
    } else {
        fft_task T = {F, a, n, 1, tw, log_threads};
        fft_rec(&T);
    }
    free(tw);
}

/* parallelize, arithmetic.rs:345-362, applied to "a[i] *= f(i)" closures */
typedef struct { const field_t *F; fe *a; size_t start, len; const fe *consts; int mode; } par_task;
static void *par_worker(void *arg) {
    par_task *T = (par_task *)arg;
    for (size_t i = 0; i < T->len; i++) {
        size_t idx = T->start + i;
        if (T->mode == 0) fe_mul(T->F, &T->a[idx], &T->a[idx], &T->consts[0]);        /* divisor */
        else { size_t r = idx % 3; if (r) fe_mul(T->F, &T->a[idx], &T->a[idx], &T->consts[r - 1]); }
    }
    return NULL;
}
static void parallelize_mul(const field_t *F, fe *a, size_t n, const fe *consts, int mode, int threads) {
    size_t chunk = n / (size_t)threads;
    if (chunk < (size_t)threads) chunk = n;
    size_t nchunks = chunk ? (n + chunk - 1) / chunk : 0;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (nchunks ? nchunks : 1));
    par_task *ts = (par_task *)malloc(sizeof(par_task) * (nchunks ? nchunks : 1));
    for (size_t c = 0; c < nchunks; c++) {
        size_t start = c * chunk, len = (start + chunk <= n) ? chunk : n - start;
        ts[c] = (par_task){F, a, start, len, consts, mode};
        if (c + 1 < nchunks) pthread_create(&th[c], NULL, par_worker, &ts[c]); else par_worker(&ts[c]);
    }
    for (size_t c = 0; c + 1 < nchunks; c++) pthread_join(th[c], NULL);
    free(th); free(ts);
}

static fe *load_vec(const field_t *F, const uint8_t *in, size_t n, size_t alloc_n) {
    fe *a = (fe *)calloc(alloc_n ? alloc_n : 1, sizeof(fe));
    for (size_t i = 0; i < n; i++) fe_from_bytes(F, &a[i], in + 32 * i);
    return a;
}
static void store_vec(const field_t *F, uint8_t *out, const fe *a, size_t n) {
    for (size_t i = 0; i < n; i++) fe_to_bytes(F, out + 32 * i, &a[i]);
}

/* best_fft(a, omega, log_n), in place on canonical bytes */
int orc_best_fft(int field, uint8_t *a, const uint8_t *omega, uint32_t log_n, int threads) {
    ensure_init(); if (threads < 1) threads = 1;
    const field_t *F = &FLD[field]; size_t n = (size_t)1 << log_n;
    fe *v = load_vec(F, a, n, n); fe w; fe_from_bytes(F, &w, omega);
    fft_mont(F, v, &w, log_n, threads);
    store_vec(F, a, v, n); free(v);
    return 0;
}
/* EvaluationDomain::ifft, domain.rs:375-383 (== lagrange_to_coeff with omega_inv, 2^-k) */
int orc_ifft(int field, uint8_t *a, const uint8_t *omega_inv, uint32_t log_n, const uint8_t *divisor, int threads) {
    ensure_init(); if (threads < 1) threads = 1;
    const field_t *F = &FLD[field]; size_t n = (size_t)1 << log_n;
    fe *v = load_vec(F, a, n, n); fe w, d; fe_from_bytes(F, &w, omega_inv); fe_from_bytes(F, &d, divisor);
    fft_mont(F, v, &w, log_n, threads);
    parallelize_mul(F, v, n, &d, 0, threads);
    store_vec(F, a, v, n); free(v);
    return 0;
}
/* coeff_to_extended, domain.rs:241-255: in = 2^k elements, out = 2^ext_k elements */
int orc_coeff_to_extended(int field, const uint8_t *in, uint32_t k, uint32_t ext_k, const uint8_t *zeta,
                          const uint8_t *ext_omega, uint8_t *out, int threads) {
    ensure_init(); if (threads < 1) threads = 1;
    const field_t *F = &FLD[field]; size_t n = (size_t)1 << k, en = (size_t)1 << ext_k;
    fe *v = load_vec(F, in, n, en); fe w, cp[2];
    fe_from_bytes(F, &w, ext_omega); fe_from_bytes(F, &cp[0], zeta); fe_sqr(F, &cp[1], &cp[0]);
    parallelize_mul(F, v, n, cp, 1, threads);          /* distribute_powers_zeta(into_coset) */
    fft_mont(F, v, &w, ext_k, threads);
    store_vec(F, out, v, en); free(v);
    return 0;
}
/* extended_to_coeff, domain.rs:303-325: in = 2^ext_k, out = out_len (= n*(j-1)) elements */
int orc_extended_to_coeff(int field, const uint8_t *in, uint32_t ext_k, const uint8_t *ext_omega_inv,
                          const uint8_t *ext_divisor, const uint8_t *zeta, size_t out_len, uint8_t *out,
                          int threads) {
    ensure_init(); if (threads < 1) threads = 1;
    const field_t *F = &FLD[field]; size_t en = (size_t)1 << ext_k;
    fe *v = load_vec(F, in, en, en); fe w, d, z, cp[2];
    fe_from_bytes(F, &w, ext_omega_inv); fe_from_bytes(F, &d, ext_divisor); fe_from_bytes(F, &z, zeta);
    fe_sqr(F, &cp[0], &z); cp[1] = z;                   /* [g_coset_inv, g_coset], domain.rs:361 */
    fft_mont(F, v, &w, ext_k, threads);
    parallelize_mul(F, v, en, &d, 0, threads);
    parallelize_mul(F, v, en, cp, 1, threads);
    store_vec(F, out, v, out_len < en ? out_len : en); free(v);
    return 0;
}

/* ---------------------------------------------------------------- best_fft with G = curve point
 * arithmetic.rs:192-295 instantiated at G = C::Curve (the FftGroup bound, :17-27): group_add / group_sub are point
 * additions, group_scale is a scalar multiplication.  Its one call site is Params::new (poly/commitment.rs:77-94):
 * g_lagrange = EC-iFFT of g, every output then scaled by 2^-k (:84-89) and batch-normalised (:91-101). */
static void scalar_mul_jac(const field_t *F, jac *r, const uint8_t k[32], const jac *base) {
    jac acc; jac_identity(F, &acc);
    for (int i = 255; i >= 0; i--) {
        jac_double(F, &acc, &acc);
        if ((k[i >> 3] >> (i & 7)) & 1) jac_add(F, &acc, &acc, base);
    }
    *r = acc;
}
static inline void jac_neg(const field_t *F, jac *r, const jac *a) { *r = *a; fe_neg(F, &r->y, &a->y); }
typedef struct { const field_t *F; jac *a; size_t n, tc; const uint8_t *tw; int depth; } ecfft_task;
static void ec_butterflies(const field_t *F, jac *left, jac *right, size_t half, size_t tc, const uint8_t *tw) {
    for (size_t i = 0; i < half; i++) {                 /* :276-293 */
        jac t = right[i], nt;
        if (i) scalar_mul_jac(F, &t, tw + 32 * (i * tc), &right[i]);
        jac_neg(F, &nt, &t);
        jac_add(F, &right[i], &left[i], &nt);
        jac_add(F, &left[i], &left[i], &t);
    }
}
static void *ecfft_rec(void *arg) {                     /* arithmetic.rs:258-295 */
    ecfft_task *T = (ecfft_task *)arg;
    if (T->n == 2) { ec_butterflies(T->F, T->a, T->a + 1, 1, T->tc, T->tw); return NULL; }
    size_t h = T->n / 2;
    ecfft_task L = {T->F, T->a, h, T->tc * 2, T->tw, T->depth - 1};
    ecfft_task R = {T->F, T->a + h, h, T->tc * 2, T->tw, T->depth - 1};
    if (T->depth > 0) {
        pthread_t th; pthread_create(&th, NULL, ecfft_rec, &L);
        ecfft_rec(&R); pthread_join(th, NULL);
    } else { ecfft_rec(&L); ecfft_rec(&R); }
    ec_butterflies(T->F, T->a, T->a + h, h, T->tc, T->tw);
    return NULL;
}
static void ecfft_core(const field_t *F, const field_t *S, jac *a, const fe *omega, uint32_t log_n, int threads) {
    size_t n = (size_t)1 << log_n;
    int log_threads = log2_floor((unsigned)threads);
    for (size_t k = 0; k < n; k++) {                    /* :207-212 */
        size_t rk = bitrev(k, log_n);
        if (k < rk) { jac t = a[k]; a[k] = a[rk]; a[rk] = t; }
    }
    size_t nt = n / 2 ? n / 2 : 1;
    uint8_t *tw = (uint8_t *)malloc(32 * nt);           /* :215-221, kept as canonical bytes (scalar-mul input) */
    fe w = S->r;
    for (size_t i = 0; i < nt; i++) { fe_to_bytes(S, tw + 32 * i, &w); fe_mul(S, &w, &w, omega); }
    if (log_n == 0) { free(tw); return; }
    if ((int)log_n <= log_threads) {
        size_t chunk = 2, tc = n / 2;
        for (uint32_t s = 0; s < log_n; s++) {
            for (size_t base = 0; base < n; base += chunk) ec_butterflies(F, a + base, a + base + chunk / 2, chunk / 2, tc, tw);
            chunk *= 2; tc /= 2;
        }
    } else {
        ecfft_task T = {F, a, n, 1, tw, log_threads};
        ecfft_rec(&T);
    }
    free(tw);
}
typedef struct { const field_t *F; jac *a; size_t len; const uint8_t *k; } ecscale_task;
static void *ecscale_worker(void *arg) {
    ecscale_task *T = (ecscale_task *)arg;
    for (size_t i = 0; i < T->len; i++) { jac t; scalar_mul_jac(T->F, &t, T->k, &T->a[i]); T->a[i] = t; }
    return NULL;
}
static void ec_scale_all(const field_t *F, jac *a, size_t n, const uint8_t *k, int threads) {   /* parallelize, :345-362 */
    size_t chunk = n / (size_t)threads;
    if (chunk < (size_t)threads) chunk = n;
    size_t nchunks = chunk ? (n + chunk - 1) / chunk : 0;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (nchunks ? nchunks : 1));
    ecscale_task *ts = (ecscale_task *)malloc(sizeof(ecscale_task) * (nchunks ? nchunks : 1));
    for (size_t c = 0; c < nchunks; c++) {
        size_t start = c * chunk, l = (start + chunk <= n) ? chunk : n - start;
        ts[c] = (ecscale_task){F, a + start, l, k};
        if (c + 1 < nchunks) pthread_create(&th[c], NULL, ecscale_worker, &ts[c]); else ecscale_worker(&ts[c]);
    }
    for (size_t c = 0; c + 1 < nchunks; c++) pthread_join(th[c], NULL);
    free(th); free(ts);
}
/* group::Curve::batch_normalize (Montgomery's trick over the non-identity z's); identity -> 64 zero bytes */
static void batch_normalize_bytes(const field_t *F, const jac *pts, size_t n, uint8_t *out) {
    fe *pre = (fe *)malloc(sizeof(fe) * (n ? n : 1)); fe acc = F->r;
    for (size_t i = 0; i < n; i++) { pre[i] = acc; if (!jac_is_id(&pts[i])) fe_mul(F, &acc, &acc, &pts[i].z); }
    fe_inv(F, &acc, &acc);
    for (size_t i = n; i-- > 0;) {
        if (jac_is_id(&pts[i])) { memset(out + 64 * i, 0, 64); continue; }
        fe zi, zi2; fe_mul(F, &zi, &acc, &pre[i]); fe_mul(F, &acc, &acc, &pts[i].z);
        fe_sqr(F, &zi2, &zi); aff r; r.inf = 0;
        fe_mul(F, &r.x, &pts[i].x, &zi2); fe_mul(F, &zi2, &zi2, &zi); fe_mul(F, &r.y, &pts[i].y, &zi2);
        aff_to_bytes(F, out + 64 * i, &r);
    }
    free(pre);
}
static jac *load_jacs(const field_t *F, const uint8_t *xyz, size_t n) {
    jac *a = (jac *)malloc(sizeof(jac) * (n ? n : 1));
    for (size_t i = 0; i < n; i++) {
        fe_from_bytes(F, &a[i].x, xyz + 96 * i); fe_from_bytes(F, &a[i].y, xyz + 96 * i + 32); fe_from_bytes(F, &a[i].z, xyz + 96 * i + 64);
    }
    return a;
}
/* in place on n = 2^log_n Jacobian points (x||y||z canonical, 96 B; z = 0 identity); scale may be NULL */
int orc_ec_fft(int curve, uint8_t *points_xyz, const uint8_t *omega, uint32_t log_n, const uint8_t *scale, int threads) {
    ensure_init();
    if (threads < 1) threads = 1;
    const field_t *F = base_field(curve), *S = scalar_field(curve);
    size_t n = (size_t)1 << log_n;
    jac *a = load_jacs(F, points_xyz, n);
    fe w; fe_from_bytes(S, &w, omega);
    ecfft_core(F, S, a, &w, log_n, threads);
    if (scale) ec_scale_all(F, a, n, scale, threads);
    for (size_t i = 0; i < n; i++) {
        fe_to_bytes(F, points_xyz + 96 * i, &a[i].x); fe_to_bytes(F, points_xyz + 96 * i + 32, &a[i].y); fe_to_bytes(F, points_xyz + 96 * i + 64, &a[i].z);
    }
    free(a);
    return 0;
}
int orc_batch_normalize(int curve, const uint8_t *points_xyz, size_t n, uint8_t *out_xy) {
    ensure_init(); const field_t *F = base_field(curve);
    jac *a = load_jacs(F, points_xyz, n);
    batch_normalize_bytes(F, a, n, out_xy);
    free(a);
    return 0;
}
/* poly/commitment.rs:74-101: g (affine) -> g_lagrange (affine).  omega_inv = alpha_inv (:77-80), minv = 2^-k (:83). */
int orc_params_lagrange(int curve, const uint8_t *g_xy, uint32_t k, const uint8_t *omega_inv, const uint8_t *minv, int threads,
                        uint8_t *out_xy) {
    ensure_init();
    if (threads < 1) threads = 1;
    const field_t *F = base_field(curve), *S = scalar_field(curve);
    size_t n = (size_t)1 << k;
    jac *a = (jac *)malloc(sizeof(jac) * n);
    for (size_t i = 0; i < n; i++) {
        aff p; aff_from_bytes(F, &p, g_xy + 64 * i);
        if (p.inf) jac_identity(F, &a[i]); else { a[i].x = p.x; a[i].y = p.y; a[i].z = F->r; }
    }
    fe w; fe_from_bytes(S, &w, omega_inv);
    ecfft_core(F, S, a, &w, k, threads);
    ec_scale_all(F, a, n, minv, threads);
    batch_normalize_bytes(F, a, n, out_xy);
    free(a);
    return 0;
}

/* ---------------------------------------------------------------- eval_polynomial / kate_division (serial in the reference)
 * arithmetic.rs:297-303 and :322-341, "TODO: parallelize?" -- restated as the same serial loops. */
int orc_eval_polynomial(int field, const uint8_t *poly, size_t n, const uint8_t *point, uint8_t *out) {
    ensure_init(); const field_t *F = &FLD[field];
    fe x, acc, c; fe_from_bytes(F, &x, point); memset(&acc, 0, sizeof acc);
    for (size_t i = n; i-- > 0;) { fe_from_bytes(F, &c, poly + 32 * i); fe_mul(F, &acc, &acc, &x); fe_add(F, &acc, &acc, &c); }
    fe_to_bytes(F, out, &acc);
    return 0;
}
int orc_kate_division(int field, const uint8_t *a, size_t n, const uint8_t *b, uint8_t *out_q) {
    ensure_init(); const field_t *F = &FLD[field];
    if (n < 2) return 0;
    fe nb, tmp, lead, r; fe_from_bytes(F, &nb, b); fe_neg(F, &nb, &nb); memset(&tmp, 0, sizeof tmp);
    for (size_t i = n - 1; i >= 1; i--) {            /* q[i-1] from a[i], :332-338 */
        fe_from_bytes(F, &r, a + 32 * i);
        fe_sub(F, &lead, &r, &tmp);
        fe_to_bytes(F, out_q + 32 * (i - 1), &lead);
        fe_mul(F, &tmp, &lead, &nb);
    }
    return 0;
}

/* ---------------------------------------------------------------- compute_s (poly/commitment/verifier.rs:156-171)
 * v[0] = init; for each challenge from the LAST to the first, the filled prefix of length len is copied behind itself and
 * the copy multiplied by u_j -- the reference's doubling loop, serial.  u: k canonical elements, out: 2^k. */
int orc_compute_s(int field, const uint8_t *u, uint32_t k, const uint8_t *init, uint8_t *out) {
    ensure_init(); const field_t *F = &FLD[field];
    if (k == 0 || k > 30) return 1;                    /* assert!(!u.is_empty()), :157 */
    size_t n = (size_t)1 << k;
    fe *v = (fe *)calloc(n, sizeof(fe)), uj;
    if (!v) return 1;
    fe_from_bytes(F, &v[0], init);
    for (uint32_t i = 0; i < k; i++) {                 /* u.iter().rev().enumerate(): len = 1 << i, u_j = u[k - 1 - i] */
        size_t len = (size_t)1 << i;
        fe_from_bytes(F, &uj, u + 32 * (size_t)(k - 1 - i));
        for (size_t t = 0; t < len; t++) fe_mul(F, &v[len + t], &v[t], &uj);
    }
    store_vec(F, out, v, n);
    free(v);
    return 0;
}

/* ---------------------------------------------------------------- the product columns and divide_by_vanishing_poly
 * Serial restatements for the tests at production sizes, where the big-integer loops of tests/grand_product_cases.py take
 * minutes.  batch_invert is ff::BatchInvert: one running product of the nonzero elements, one inversion, a backward sweep;
 * zeros stay zero.  Returns 1 when its scratch cannot be allocated. */
static int batch_invert(const field_t *F, fe *a, size_t n) {
    fe *pre = (fe *)malloc((n ? n : 1) * sizeof(fe)), acc, t;
    if (!pre) return 1;
    fe_from_bytes(F, &acc, (const uint8_t[32]){1});
    for (size_t i = 0; i < n; i++) {
        pre[i] = acc;
        if (!fe_is_zero(&a[i])) fe_mul(F, &acc, &acc, &a[i]);
    }
    fe_inv(F, &acc, &acc);
    for (size_t i = n; i-- > 0;) {
        if (fe_is_zero(&a[i])) continue;
        fe_mul(F, &t, &acc, &pre[i]);                   /* a[i]^-1 = (a[0..i] product)^-1 * (a[0..i-1] product) */
        fe_mul(F, &acc, &acc, &a[i]);
        a[i] = t;
    }
    free(pre);
    return 0;
}
/* permutation::Argument::commit, plonk/permutation/prover.rs:81-168, for `proofs` proofs of the same sigmas.  columns:
 * proofs x cols x n, sigmas: cols x n, blinding: proofs x sets x bf values in the rng's order, out: proofs x sets x n. */
int orc_permutation_product(int field, const uint8_t *columns, const uint8_t *sigmas, size_t proofs, size_t cols, size_t chunk_len, uint32_t k,
                            const uint8_t *beta, const uint8_t *gamma, const uint8_t *omega, const uint8_t *delta, const uint8_t *blinding,
                            uint32_t bf, uint8_t *out) {
    ensure_init(); const field_t *F = &FLD[field];
    const size_t n = (size_t)1 << k;
    if (chunk_len == 0 || (size_t)bf + 1 >= n) return 1;
    fe b, g, w, d, one, x, y;
    fe_from_bytes(F, &b, beta); fe_from_bytes(F, &g, gamma); fe_from_bytes(F, &w, omega); fe_from_bytes(F, &d, delta);
    fe_from_bytes(F, &one, (const uint8_t[32]){1});
    fe *mv = (fe *)malloc(n * sizeof(fe));
    if (!mv) return 1;
    size_t set_at = 0;
    for (size_t p = 0; p < proofs; p++) {
        fe last_z = one, deltaomega = one;
        for (size_t c0 = 0; c0 < cols; c0 += chunk_len, set_at++) {
            const size_t c1 = c0 + chunk_len < cols ? c0 + chunk_len : cols;
            for (size_t i = 0; i < n; i++) mv[i] = one;
            for (size_t c = c0; c < c1; c++) {                                  /* :101-116, v + beta sigma + gamma */
                const uint8_t *v = columns + 32 * n * (p * cols + c), *s = sigmas + 32 * n * c;
                for (size_t i = 0; i < n; i++) {
                    fe_from_bytes(F, &x, s + 32 * i); fe_mul(F, &x, &x, &b); fe_add(F, &x, &x, &g);
                    fe_from_bytes(F, &y, v + 32 * i); fe_add(F, &x, &x, &y);
                    fe_mul(F, &mv[i], &mv[i], &x);
                }
            }
            if (batch_invert(F, mv, n)) { free(mv); return 1; }                 /* :120 */
            for (size_t c = c0; c < c1; c++) {                                  /* :124-143, v + delta^j omega^i beta + gamma */
                const uint8_t *v = columns + 32 * n * (p * cols + c);
                fe cur = deltaomega;
                for (size_t i = 0; i < n; i++) {
                    fe_mul(F, &x, &cur, &b); fe_add(F, &x, &x, &g);
                    fe_from_bytes(F, &y, v + 32 * i); fe_add(F, &x, &x, &y);
                    fe_mul(F, &mv[i], &mv[i], &x);
                    fe_mul(F, &cur, &cur, &w);
                }
                fe_mul(F, &deltaomega, &deltaomega, &d);
            }
            uint8_t *z = out + 32 * n * set_at;                                 /* :150-156, z[0] = last_z */
            fe acc = last_z;
            for (size_t i = 0; i < n; i++) {
                if (i == n - bf - 1) last_z = acc;                              /* :163 */
                fe_to_bytes(F, z + 32 * i, &acc);
                fe_mul(F, &acc, &acc, &mv[i]);
            }
            if (bf) memcpy(z + 32 * (n - bf), blinding + 32 * (size_t)bf * set_at, 32 * (size_t)bf);   /* :158-161 */
        }
    }
    free(mv);
    return 0;
}
/* lookup::Permuted::commit_product, plonk/lookup/prover.rs:279-321, for one lookup: the compressed input and table a, s, the
 * permuted a', s' (n each), bf blinding values; out: n. */
int orc_lookup_product(int field, const uint8_t *a, const uint8_t *s, const uint8_t *a_perm, const uint8_t *s_perm, uint32_t k, const uint8_t *beta,
                       const uint8_t *gamma, const uint8_t *blinding, uint32_t bf, uint8_t *out) {
    ensure_init(); const field_t *F = &FLD[field];
    const size_t n = (size_t)1 << k;
    if ((size_t)bf + 1 >= n) return 1;
    fe b, g, x, y;
    fe_from_bytes(F, &b, beta); fe_from_bytes(F, &g, gamma);
    fe *lp = (fe *)malloc(n * sizeof(fe));
    if (!lp) return 1;
    for (size_t i = 0; i < n; i++) {                                           /* :281-291 */
        fe_from_bytes(F, &x, a_perm + 32 * i); fe_add(F, &x, &x, &b);
        fe_from_bytes(F, &y, s_perm + 32 * i); fe_add(F, &y, &y, &g);
        fe_mul(F, &lp[i], &x, &y);
    }
    if (batch_invert(F, lp, n)) { free(lp); return 1; }                        /* :295 */
    for (size_t i = 0; i < n; i++) {                                           /* :299-309 */
        fe_from_bytes(F, &x, a + 32 * i); fe_add(F, &x, &x, &b); fe_mul(F, &lp[i], &lp[i], &x);
        fe_from_bytes(F, &y, s + 32 * i); fe_add(F, &y, &y, &g); fe_mul(F, &lp[i], &lp[i], &y);
    }
    fe acc; fe_from_bytes(F, &acc, (const uint8_t[32]){1});                    /* :311-318, z[0] = ONE */
    for (size_t i = 0; i < n - bf; i++) {
        fe_to_bytes(F, out + 32 * i, &acc);
        fe_mul(F, &acc, &acc, &lp[i]);
    }
    if (bf) memcpy(out + 32 * (n - bf), blinding, 32 * (size_t)bf);            /* :319-321 */
    free(lp);
    return 0;
}
/* divide_by_vanishing_poly, poly/domain.rs:329-348: a[i] *= t_evaluations[i % t_len], in place on len canonical elements */
int orc_divide_by_vanishing_poly(int field, uint8_t *a, size_t len, const uint8_t *t_evals, size_t t_len) {
    ensure_init(); const field_t *F = &FLD[field];
    if (t_len == 0) return 1;
    fe x, t;
    for (size_t i = 0; i < len; i++) {
        fe_from_bytes(F, &x, a + 32 * i); fe_from_bytes(F, &t, t_evals + 32 * (i % t_len));
        fe_mul(F, &x, &x, &t); fe_to_bytes(F, a + 32 * i, &x);
    }
    return 0;
}

/* ---------------------------------------------------------------- permute_expression_pair (plonk/lookup/prover.rs:563-647)
 * The usable rows only (the blinding rows, :625-627, are random).  Serial like the reference: sort the input (:577-581); the
 * reference's BTreeMap of table values with counts (:584-591) is restated as the sorted table with one "taken" mark per value
 * consumed -- iterating what is left in ascending order is the map's iteration order (:617); repeated rows are handed out
 * from the back (:619, `pop`).  Canonical 32-byte little-endian values in and out.  Returns 1 where the reference returns
 * Error::ConstraintSystemFailure (:605-608). */
static int cmp_bytes32(const void *a, const void *b) {
    const uint8_t *x = (const uint8_t *)a, *y = (const uint8_t *)b;
    for (int i = 31; i >= 0; i--) if (x[i] != y[i]) return x[i] < y[i] ? -1 : 1;
    return 0;
}
int orc_permute_expression_pair(const uint8_t *input, const uint8_t *table, size_t usable_rows, uint8_t *out_input, uint8_t *out_table) {
    const size_t u = usable_rows;
    if (u == 0) return 0;
    uint8_t *ts = (uint8_t *)malloc(32 * u), *taken = (uint8_t *)calloc(u, 1);
    size_t *rep = (size_t *)malloc(sizeof(size_t) * u), nrep = 0;
    memcpy(out_input, input, 32 * u); qsort(out_input, u, 32, cmp_bytes32);
    memcpy(ts, table, 32 * u); qsort(ts, u, 32, cmp_bytes32);
    int rc = 0;
    for (size_t row = 0; row < u && !rc; row++) {
        const uint8_t *v = out_input + 32 * row;
        if (row == 0 || cmp_bytes32(v, v - 32) != 0) {
            memcpy(out_table + 32 * row, v, 32);
            size_t lo = 0, hi = u;                       /* first instance of v in the sorted table */
            while (lo < hi) { size_t mid = (lo + hi) / 2; if (cmp_bytes32(ts + 32 * mid, v) < 0) lo = mid + 1; else hi = mid; }
            if (lo >= u || cmp_bytes32(ts + 32 * lo, v) != 0) rc = 1; else taken[lo] = 1;
        } else rep[nrep++] = row;
    }
    for (size_t i = 0; i < u && !rc; i++)
        if (!taken[i]) memcpy(out_table + 32 * rep[--nrep], ts + 32 * i, 32);
    free(ts); free(taken); free(rep);
    return rc;
}

/* ---------------------------------------------------------------- Evaluator::evaluate (poly/evaluator.rs:129-228)
 * The Ast arrives flattened in postfix form (four uint32 per instruction: op, arg, shift, 0 -- 0 POLY, 1 CONST, 2 LINEAR, 3 ADD,
 * 4 MUL, 5 SCALE, 6 NEG; DistributePowers = CONST 0 then SCALE base / term / ADD per term); like the reference the work is split
 * into chunks of elements, one thread each (multicore::scope, :199-216).  Used as the timed CPU baseline of the quotient pipeline. */
typedef struct { const field_t *F; const fe *const *polys; const uint32_t *code; uint32_t n_code; const fe *consts; fe lin0, omega; uint64_t n, lo, hi; fe *out; } ast_task;
static void *ast_worker(void *arg) {
    ast_task *T = (ast_task *)arg; const field_t *F = T->F;
    fe st[32], lin; uint64_t e[4] = {T->lo, 0, 0, 0};
    fe_pow(F, &lin, &T->omega, e); fe_mul(F, &lin, &lin, &T->lin0);        /* lin_base * omega^lo, :545-553 */
    for (uint64_t i = T->lo; i < T->hi; i++) {
        uint32_t sp = 0;
        for (uint32_t pc = 0; pc < T->n_code; pc++) {
            const uint32_t *in = T->code + 4 * pc;
            switch (in[0]) {
            case 0: st[sp++] = T->polys[in[1]][(i + (uint64_t)(int64_t)(int32_t)in[2]) & (T->n - 1)]; break;
            case 1: st[sp++] = T->consts[in[1]]; break;
            case 2: fe_mul(F, &st[sp], &lin, &T->consts[in[1]]); sp++; break;
            case 3: sp--; fe_add(F, &st[sp - 1], &st[sp - 1], &st[sp]); break;
            case 4: sp--; fe_mul(F, &st[sp - 1], &st[sp - 1], &st[sp]); break;
            case 5: fe_mul(F, &st[sp - 1], &st[sp - 1], &T->consts[in[1]]); break;
            default: fe_neg(F, &st[sp - 1], &st[sp - 1]); break;
            }
        }
        T->out[i] = st[0];
        fe_mul(F, &lin, &lin, &T->omega);
    }
    return NULL;
}
int orc_ast_eval(int field, const uint8_t *polys, uint32_t n_polys, uint32_t log_n, const uint32_t *code, uint32_t n_code, const uint8_t *consts,
                 uint32_t n_consts, const uint8_t *omega, const uint8_t *lin_base, int threads, uint8_t *out) {
    ensure_init(); const field_t *F = &FLD[field];
    if (threads < 1) threads = 1;
    uint64_t n = (uint64_t)1 << log_n;
    fe **pp = (fe **)malloc(sizeof(fe *) * (n_polys ? n_polys : 1));
    for (uint32_t b = 0; b < n_polys; b++) pp[b] = load_vec(F, polys + 32 * n * b, n, n);
    fe *cs = load_vec(F, consts, n_consts, n_consts ? n_consts : 1), *o = (fe *)malloc(sizeof(fe) * n);
    fe w, l0; fe_from_bytes(F, &w, omega); fe_from_bytes(F, &l0, lin_base);
    uint64_t chunks = (uint64_t)threads * 4, cs_len = (n + chunks - 1) / chunks;       /* get_chunk_params, :16-32 */
    uint64_t nch = (n + cs_len - 1) / cs_len;
    ast_task *ts = (ast_task *)malloc(sizeof(ast_task) * nch); pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * nch);
    for (uint64_t c = 0; c < nch; c++) {
        uint64_t lo = c * cs_len, hi = lo + cs_len < n ? lo + cs_len : n;
        ts[c] = (ast_task){F, (const fe *const *)pp, code, n_code, cs, l0, w, n, lo, hi, o};
        if (c + 1 < nch) pthread_create(&th[c], NULL, ast_worker, &ts[c]); else ast_worker(&ts[c]);
    }
    for (uint64_t c = 0; c + 1 < nch; c++) pthread_join(th[c], NULL);
    store_vec(F, out, o, n);
    for (uint32_t b = 0; b < n_polys; b++) free(pp[b]);
    free(pp); free(cs); free(o); free(ts); free(th);
    return 0;
}

/* ---------------------------------------------------------------- field / curve primitives for KATs */
/* op: 0 add, 1 sub, 2 mul, 3 inv(a), 4 a^5, 5 neg(a) */
int orc_field_op(int field, int op, const uint8_t *a, const uint8_t *b, uint8_t *out) {
    ensure_init();
    const field_t *F = &FLD[field]; fe x, y, r;
    fe_from_bytes(F, &x, a); if (b) fe_from_bytes(F, &y, b); else y = F->r;
    switch (op) {
    case 0: fe_add(F, &r, &x, &y); break;
    case 1: fe_sub(F, &r, &x, &y); break;
    case 2: fe_mul(F, &r, &x, &y); break;
    case 3: fe_inv(F, &r, &x); break;
    case 4: fe_sqr(F, &r, &x); fe_sqr(F, &r, &r); fe_mul(F, &r, &r, &x); break;
    case 5: fe_neg(F, &r, &x); break;
    default: return -1;
    }
    fe_to_bytes(F, out, &r);
    return 0;
}
int orc_scalar_mul(int curve, const uint8_t *scalar, const uint8_t *base_xy, uint8_t *out_xy) {
    ensure_init(); const field_t *F = base_field(curve);
    aff b, r; aff_from_bytes(F, &b, base_xy);
    jac t; scalar_mul_bytes(F, &t, scalar, &b);
    jac_to_aff(F, &r, &t); aff_to_bytes(F, out_xy, &r);
    return 0;
}
int orc_point_add(int curve, const uint8_t *a_xy, const uint8_t *b_xy, uint8_t *out_xy) {
    ensure_init(); const field_t *F = base_field(curve);
    aff a, b, r; aff_from_bytes(F, &a, a_xy); aff_from_bytes(F, &b, b_xy);
    jac t; if (a.inf) jac_identity(F, &t); else { t.x = a.x; t.y = a.y; t.z = F->r; }
    jac_add_mixed(F, &t, &t, &b);
    jac_to_aff(F, &r, &t); aff_to_bytes(F, out_xy, &r);
    return 0;
}
/* Jacobian (x,y,z canonical bytes, 96 B) -> affine 64 B */
int orc_jac_to_affine(int curve, const uint8_t *xyz, uint8_t *out_xy) {
    ensure_init(); const field_t *F = base_field(curve);
    jac t; fe_from_bytes(F, &t.x, xyz); fe_from_bytes(F, &t.y, xyz + 32); fe_from_bytes(F, &t.z, xyz + 64);
    aff r; jac_to_aff(F, &r, &t); aff_to_bytes(F, out_xy, &r);
    return 0;
}
int orc_on_curve(int curve, const uint8_t *xy) {
    ensure_init(); const field_t *F = base_field(curve);
    aff a; aff_from_bytes(F, &a, xy); if (a.inf) return 1;
    fe l, r, five, t; fe_sqr(F, &l, &a.y); fe_sqr(F, &r, &a.x); fe_mul(F, &r, &r, &a.x);
    uint8_t fb[32] = {5}; fe_from_bytes(F, &five, fb); fe_add(F, &r, &r, &five);
    (void)t; return fe_eq(&l, &r);
}

/* ---------------------------------------------------------------- seeded inputs (same PRNG as pasta.py) */
typedef struct { uint64_t s[4]; } xo_t;
static inline uint64_t rotl64(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
static void xo_seed(xo_t *x, uint64_t seed) {
    for (int i = 0; i < 4; i++) {
        seed += 0x9E3779B97F4A7C15ULL; uint64_t z = seed;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
        x->s[i] = z ^ (z >> 31);
    }
}
static uint64_t xo_next(xo_t *x) {
    uint64_t *s = x->s, result = rotl64(s[1] * 5, 7) * 9, t = s[1] << 17;
    s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t; s[3] = rotl64(s[3], 45);
    return result;
}
static void xo_field(xo_t *x, const field_t *F, uint8_t out[32]) {
    uint64_t v[4];
    do { for (int i = 0; i < 4; i++) v[i] = xo_next(x); v[3] &= 0x7fffffffffffffffULL; } while (ge4(v, F->m));
    memcpy(out, v, 32);
}
int orc_gen_scalars(int field, uint64_t seed, size_t n, uint8_t *out) {
    ensure_init(); xo_t x; xo_seed(&x, seed);
    for (size_t i = 0; i < n; i++) xo_field(&x, &FLD[field], out + 32 * i);
    return 0;
}
/* P_0 = [s]G, P_{i+1} = P_i + [t]G, G = (-1, 2); batch-normalised */
int orc_gen_points(int curve, uint64_t seed, size_t n, uint8_t *out) {
    ensure_init(); const field_t *F = base_field(curve), *S = scalar_field(curve);
    xo_t x; xo_seed(&x, seed);
    uint8_t sb[32], tb[32]; xo_field(&x, S, sb); xo_field(&x, S, tb);
    aff g; fe one = F->r, two; fe_neg(F, &g.x, &one); fe_add(F, &two, &one, &one); g.y = two; g.inf = 0;
    jac cur, step; scalar_mul_bytes(F, &cur, sb, &g); scalar_mul_bytes(F, &step, tb, &g);
    jac *pts = (jac *)malloc(sizeof(jac) * (n ? n : 1));
    for (size_t i = 0; i < n; i++) { pts[i] = cur; jac_add(F, &cur, &cur, &step); }
    /* Montgomery-trick batch normalisation */
    fe *pre = (fe *)malloc(sizeof(fe) * (n ? n : 1)); fe acc = F->r;
    for (size_t i = 0; i < n; i++) { pre[i] = acc; if (!jac_is_id(&pts[i])) fe_mul(F, &acc, &acc, &pts[i].z); }
    fe_inv(F, &acc, &acc);
    for (size_t i = n; i-- > 0;) {
        if (jac_is_id(&pts[i])) { memset(out + 64 * i, 0, 64); continue; }
        fe zi, zi2; fe_mul(F, &zi, &acc, &pre[i]); fe_mul(F, &acc, &acc, &pts[i].z);
        fe_sqr(F, &zi2, &zi); aff r; r.inf = 0;
        fe_mul(F, &r.x, &pts[i].x, &zi2); fe_mul(F, &zi2, &zi2, &zi); fe_mul(F, &r.y, &pts[i].y, &zi2);
        aff_to_bytes(F, out + 64 * i, &r);
    }
    free(pts); free(pre);
    return 0;
}

/* ---------------------------------------------------------------- IPA round loop
 * poly/commitment/prover.rs:100-142 with the transcript factored out (challenges and randomness are
 * inputs).  bases: g[0..n) || w || u (canonical affine).  Outputs: L_j, R_j affine (k x 64 B each), c (32 B). */
typedef struct { const field_t *F; aff *lo; const aff *hi; size_t len; const uint8_t *u; } collapse_task;
static void *collapse_worker(void *arg) {              /* prover.rs:158-165: one parallelize chunk */
    collapse_task *T = (collapse_task *)arg;
    const field_t *F = T->F;
    size_t len = T->len;
    jac *tmp = (jac *)malloc(sizeof(jac) * (len ? len : 1));
    fe *pre = (fe *)malloc(sizeof(fe) * (len ? len : 1));
    for (size_t i = 0; i < len; i++) {
        jac t; scalar_mul_bytes(F, &t, T->u, &T->hi[i]);
        jac_add_mixed(F, &tmp[i], &t, &T->lo[i]);
    }
    /* batch_normalize: Montgomery's trick over the non-identity z's */
    fe acc = F->r;
    for (size_t i = 0; i < len; i++) { pre[i] = acc; if (!jac_is_id(&tmp[i])) fe_mul(F, &acc, &acc, &tmp[i].z); }
    fe inv; fe_inv(F, &inv, &acc);
    for (size_t i = len; i-- > 0;) {
        if (jac_is_id(&tmp[i])) { memset(&T->lo[i], 0, sizeof(aff)); T->lo[i].inf = 1; continue; }
        fe zi, zi2; fe_mul(F, &zi, &inv, &pre[i]); fe_mul(F, &inv, &inv, &tmp[i].z);
        fe_sqr(F, &zi2, &zi);
        fe_mul(F, &T->lo[i].x, &tmp[i].x, &zi2); fe_mul(F, &zi2, &zi2, &zi); fe_mul(F, &T->lo[i].y, &tmp[i].y, &zi2);
        T->lo[i].inf = 0;
    }
    free(tmp); free(pre);
    return NULL;
}
static void generator_collapse(const field_t *F, aff *g, size_t len, const uint8_t *u, int threads) {
    size_t half = len / 2, chunk = half / (size_t)threads;
    if (chunk < (size_t)threads) chunk = half;          /* arithmetic.rs:347-351 */
    size_t nchunks = chunk ? (half + chunk - 1) / chunk : 0;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (nchunks ? nchunks : 1));
    collapse_task *ts = (collapse_task *)malloc(sizeof(collapse_task) * (nchunks ? nchunks : 1));
    for (size_t c = 0; c < nchunks; c++) {
        size_t start = c * chunk, l = (start + chunk <= half) ? chunk : half - start;
        ts[c] = (collapse_task){F, g + start, g + half + start, l, u};
        if (c + 1 < nchunks) pthread_create(&th[c], NULL, collapse_worker, &ts[c]); else collapse_worker(&ts[c]);
    }
    for (size_t c = 0; c + 1 < nchunks; c++) pthread_join(th[c], NULL);
    free(th); free(ts);
}
/* challenge source of the transcript-driven form: called once per round with the affine L_j, R_j just computed
 * (prover.rs:124-128 writes them to the transcript and squeezes u_j); writes the canonical u_j */
typedef void (*orc_challenge_fn)(uint32_t j, const uint8_t *l_xy, const uint8_t *r_xy, uint8_t *u_out, void *ctx);
static int ipa_rounds_impl(int curve, const uint8_t *bases, uint32_t k, const uint8_t *p_prime, const uint8_t *x3, const uint8_t *z,
                           const uint8_t *challenges, orc_challenge_fn cb, void *cb_ctx, const uint8_t *l_rand, const uint8_t *r_rand, int threads,
                           uint8_t *out_l_xy, uint8_t *out_r_xy, uint8_t *out_c);
int orc_ipa_rounds(int curve, const uint8_t *bases, uint32_t k, const uint8_t *p_prime, const uint8_t *x3, const uint8_t *z,
                   const uint8_t *challenges, const uint8_t *l_rand, const uint8_t *r_rand, int threads,
                   uint8_t *out_l_xy, uint8_t *out_r_xy, uint8_t *out_c) {
    return ipa_rounds_impl(curve, bases, k, p_prime, x3, z, challenges, NULL, NULL, l_rand, r_rand, threads, out_l_xy, out_r_xy, out_c);
}
int orc_ipa_rounds_cb(int curve, const uint8_t *bases, uint32_t k, const uint8_t *p_prime, const uint8_t *x3, const uint8_t *z,
                      orc_challenge_fn cb, void *cb_ctx, const uint8_t *l_rand, const uint8_t *r_rand, int threads,
                      uint8_t *out_l_xy, uint8_t *out_r_xy, uint8_t *out_c) {
    return ipa_rounds_impl(curve, bases, k, p_prime, x3, z, NULL, cb, cb_ctx, l_rand, r_rand, threads, out_l_xy, out_r_xy, out_c);
}
static int ipa_rounds_impl(int curve, const uint8_t *bases, uint32_t k, const uint8_t *p_prime, const uint8_t *x3, const uint8_t *z,
                           const uint8_t *challenges, orc_challenge_fn cb, void *cb_ctx, const uint8_t *l_rand, const uint8_t *r_rand, int threads,
                           uint8_t *out_l_xy, uint8_t *out_r_xy, uint8_t *out_c) {
    ensure_init();
    if (threads < 1) threads = 1;
    const field_t *F = base_field(curve), *S = scalar_field(curve);
    size_t n = (size_t)1 << k;
    aff *g = (aff *)malloc(sizeof(aff) * n), wu[2];
    for (size_t i = 0; i < n; i++) aff_from_bytes(F, &g[i], bases + 64 * i);
    aff_from_bytes(F, &wu[1], bases + 64 * n);           /* [u, w] order of prover.rs:118 */
    aff_from_bytes(F, &wu[0], bases + 64 * (n + 1));
    fe *p = load_vec(S, p_prime, n, n), *b = (fe *)malloc(sizeof(fe) * n);
    fe x, zz; fe_from_bytes(S, &x, x3); fe_from_bytes(S, &zz, z);
    fe cur = S->r;
    for (size_t i = 0; i < n; i++) { b[i] = cur; fe_mul(S, &cur, &cur, &x); }      /* :86-93 */
    uint8_t *sc = (uint8_t *)malloc(32 * n);
    for (uint32_t j = 0; j < k; j++) {
        size_t half = (size_t)1 << (k - j - 1);
        jac lj, rj, t;
        store_vec(S, sc, p + half, half); msm_core(F, sc, g, half, threads, &lj);            /* :107 */
        store_vec(S, sc, p, half); msm_core(F, sc, g + half, half, threads, &rj);            /* :108 */
        fe vl, vr, m; memset(&vl, 0, sizeof vl); memset(&vr, 0, sizeof vr);
        for (size_t i = 0; i < half; i++) {                                                  /* :110-111 */
            fe_mul(S, &m, &p[i + half], &b[i]); fe_add(S, &vl, &vl, &m);
            fe_mul(S, &m, &p[i], &b[i + half]); fe_add(S, &vr, &vr, &m);
        }
        uint8_t two[64];
        fe_mul(S, &m, &vl, &zz); fe_to_bytes(S, two, &m); memcpy(two + 32, l_rand + 32 * j, 32);
        msm_core(F, two, wu, 2, threads, &t); jac_add(F, &lj, &lj, &t);                      /* :118 */
        fe_mul(S, &m, &vr, &zz); fe_to_bytes(S, two, &m); memcpy(two + 32, r_rand + 32 * j, 32);
        msm_core(F, two, wu, 2, threads, &t); jac_add(F, &rj, &rj, &t);                      /* :119 */
        aff a; jac_to_aff(F, &a, &lj); aff_to_bytes(F, out_l_xy + 64 * j, &a);
        jac_to_aff(F, &a, &rj); aff_to_bytes(F, out_r_xy + 64 * j, &a);
        uint8_t ub[32];
        if (cb) cb(j, out_l_xy + 64 * j, out_r_xy + 64 * j, ub, cb_ctx); else memcpy(ub, challenges + 32 * j, 32);
        fe u, ui; fe_from_bytes(S, &u, ub); fe_inv(S, &ui, &u);
        for (size_t i = 0; i < half; i++) {                                                  /* :134-137 */
            fe_mul(S, &m, &p[i + half], &ui); fe_add(S, &p[i], &p[i], &m);
            fe_mul(S, &m, &b[i + half], &u); fe_add(S, &b[i], &b[i], &m);
        }
        generator_collapse(F, g, 2 * half, ub, threads);                                     /* :140 */
    }
    fe_to_bytes(S, out_c, &p[0]);
    free(g); free(p); free(b); free(sc);
    return 0;
}
