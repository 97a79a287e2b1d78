// C ABI of the engine, part 5 of 5: reductions and elementwise programs on resident polynomials (polyops.cuh, asteval.cuh),
// the lookup permutation (lookup.cuh), the verifier's MSM scalars (verifier.cuh), the permutation polynomials (keygen.cuh),
// their copy cycles (assembly.cuh) and the permutation / lookup product columns (grandproduct.cuh).
#include "util_kernels.cuh"
#include "polyops.cuh"
#include "asteval.cuh"
#include "lookup.cuh"
#include "verifier.cuh"
#include "keygen.cuh"
#include "assembly.cuh"
#include "grandproduct.cuh"
#include "chacha.cuh"

// ------------------------------------------------------------------------------------------------
// eval_polynomial / compute_inner_product / kate_division on resident polynomials (polyops.cuh)
// ------------------------------------------------------------------------------------------------
// mode 0: eval (points: batch x 32 host), 1: inner product of a[i] and c[i], 2: kate division of a[i] by (X - point_i) into c[i]
template <class P>
static int polyops_run(int mode, const std::vector<PolyBuf *> &a, const std::vector<PolyBuf *> &c, size_t n, const void *points, const HostArgs &h,
                       void *out) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint32_t batch = (uint32_t)a.size();
    GpTree T;
    if (const char *e = gp_reduce_plan(n, batch, mode == 1, &T)) return fail(std::string(h.who) + ": " + e);
    const uint64_t *m = T.m;
    const size_t L = T.L;                                        // levels above the polynomial itself
    if (X.po_lvl.ensure(T.total * sizeof(fe)) || X.po_q.ensure(T.total * sizeof(fe)) || X.po_pts.ensure((L + 2) * batch * sizeof(fe)) ||
        X.misc.ensure(batch * sizeof(fe) + 64))
        return 1;
    fe *lvl = X.po_lvl.as<fe>(), *qarr = X.po_q.as<fe>(), *pts = X.po_pts.as<fe>();
    auto level = [&](size_t l) { return lvl + T.off[l]; };       // values of level l >= 1: [batch][m[l]]
    auto qlevel = [&](size_t l) { return qarr + T.off[l]; };
    std::vector<PolyBuf *> cols(a);                              // a, then c (null pointers without it)
    cols.insert(cols.end(), c.begin(), c.end());
    cols.resize(2 * batch);
    ColTable t;
    if (col_table(cols, nullptr, 0, s, &t)) return 1;
    const fe *const *d_a = t.cols;
    fe *const *d_c = t.cols + batch;
    // points of level 0 (Montgomery): the caller's, or 1 for the plain sums of the inner product
    if (mode == 1) {
        LAUNCH(fe_fill_kernel<P>, blocks_for(batch, 64), 64, 0, s, pts, batch, fe_one<P>());
    } else if (h.up(P::ID, pts, points, batch, s)) {
        return 1;
    }
    if (mode != 1 && n <= (1ull << 16) && n >= 2 && X.poly_cta) {
        // small polynomials: one CTA per polynomial does the whole reduction (polyops.cuh poly_eval_cta_kernel / poly_kate_cta_kernel)
        if (mode == 0) {
            fe *res = X.misc.as<fe>();
            LAUNCH(poly_eval_cta_kernel<P>, batch, H2_POLY_CTA, 0, s, d_a, (uint64_t)n, (const fe *)pts, res);
            if (h.from_mont(P::ID, res, batch, s)) return 1;
            CU(cudaMemcpyAsync(out, res, batch * sizeof(fe), cudaMemcpyDeviceToHost, s));
            CU(cudaStreamSynchronize(s));
            return 0;
        }
        LAUNCH(poly_kate_cta_kernel<P>, batch, H2_KATE_CTA, 0, s, d_a, (uint64_t)n, (const fe *)pts, d_c);
        for (uint32_t b = 0; b < batch; b++) CU(cudaMemsetAsync(c[b]->buf.as<fe>() + (n - 1), 0, sizeof(fe), s));
        return 0;
    }
    // upward pass: level l + 1 from level l at the point x^(CHUNK^l)
    for (size_t l = 0; l < L; l++) {
        const dim3 grid(blocks_for(m[l + 1], 128), batch);
        if (l == 0 && mode == 1) LAUNCH(poly_inner_level0_kernel<P>, grid, 128, 0, s, d_a, d_c, m[0], level(1), m[1]);
        else LAUNCH(poly_eval_level_kernel<P>, grid, 128, 0, s, l == 0 ? d_a : (const fe *const *)nullptr, l == 0 ? (const fe *)nullptr : (const fe *)level(l),
                    m[l], (const fe *)(pts + l * batch), level(l + 1), m[l + 1]);
        if (mode != 1) LAUNCH(poly_pow_chunk_kernel<P>, blocks_for(batch, 64), 64, 0, s, (const fe *)(pts + l * batch), pts + (l + 1) * batch, batch);
        else if (l == 0) LAUNCH(fe_fill_kernel<P>, blocks_for(batch, 64), 64, 0, s, pts + batch, batch, fe_one<P>());
        if (mode == 1 && l >= 1) CU(cudaMemcpyAsync(pts + (l + 1) * batch, pts, batch * sizeof(fe), cudaMemcpyDeviceToDevice, s));
    }
    if (mode != 2) {   // the single value of the top level is the result (n == 1: the coefficient itself; n == 0 handled by the caller)
        fe *res = X.misc.as<fe>();
        if (L == 0) {
            for (uint32_t b = 0; b < batch; b++) CU(cudaMemcpyAsync(res + b, a[b]->buf.as<fe>(), sizeof(fe), cudaMemcpyDeviceToDevice, s));
        } else {
            CU(cudaMemcpyAsync(res, level(L), batch * sizeof(fe), cudaMemcpyDeviceToDevice, s));   // m[L] == 1: [batch][1]
        }
        if (h.from_mont(P::ID, res, batch, s)) return 1;
        CU(cudaMemcpyAsync(out, res, batch * sizeof(fe), cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        return 0;
    }
    // kate division, downward pass: Q at every position of level l from the carries of level l + 1.  The top level with
    // more than one value (m[L] == 1 always; start from the highest level that has something to walk) needs no carry.
    for (size_t l = L; l-- > 0;) {
        const dim3 grid(blocks_for(m[l + 1], 128), batch);
        const fe *carry = (l + 1 < L) ? (const fe *)qlevel(l + 1) : (const fe *)nullptr;   // Q of level l + 1; the top level's Q(1..) are zero
        LAUNCH(poly_kate_down_kernel<P>, grid, 128, 0, s, l == 0 ? d_a : (const fe *const *)nullptr, l == 0 ? (const fe *)nullptr : (const fe *)level(l), m[l],
               (const fe *)(pts + l * batch), carry, m[l + 1], l == 0 ? (fe *)nullptr : qlevel(l), l == 0 ? d_c : (fe *const *)nullptr);
    }
    // the quotient has n - 1 coefficients; slot n - 1 becomes the zero the reference pushes before committing n of them
    // (poly/multiopen/prover.rs: `kate_division(..); poly.push(ZERO)`)
    for (uint32_t b = 0; b < batch; b++) CU(cudaMemsetAsync(c[b]->buf.as<fe>() + (n - 1), 0, sizeof(fe), s));
    return 0;
}
// h: checked by the caller
static int polyops_dispatch(int mode, const uint64_t *ah, const uint64_t *ch, size_t batch, size_t n, const void *points, const HostArgs &h, void *out) {
    const char *who = h.who;
    CtxLock lk;
    if (require_ready()) return 1;
    if (batch == 0) return 0;
    if (batch > 256) return fail(std::string(who) + ": batch > 256");
    if (n >= (1ull << 32)) return fail(std::string(who) + ": n >= 2^32");
    PolyArgs g(who);
    std::vector<PolyBuf *> a, c;
    if (mode == 2) {   // kate division writes quotients of n - 1 coefficients; the inner product reads both operands
        if (g.out(ch, batch, "dst", n - 1, "n - 1", c) || g.in(ah, batch, "src", n, "n", a) || g.distinct()) return 1;
    } else if (g.in(ah, batch, mode == 0 ? "polys" : "a", n, "n", a) || (ch && g.in(ch, batch, "b", n, "n", c))) {
        return 1;
    }
    return by_field(a[0]->field, [&](auto p) { return polyops_run<decltype(p)>(mode, a, c, n, points, h, out); });
}
// Evaluator::evaluate (poly/evaluator.rs:129-228) on resident polynomials: `code` is the postfix form of the Ast (asteval.cuh),
// validated here so that the kernel's operand stack can neither overflow nor underflow.
template <class P>
static int ast_run(PolyBuf *out, const std::vector<PolyBuf *> &polys, uint32_t log_n, const AstInstr *code, size_t n_code, const void *consts,
                   size_t n_consts, const void *omega, const void *lin_base, const HostArgs &h, bool has_linear) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint64_t n = 1ull << log_n;
    if (X.ast_code.ensure(n_code * sizeof(AstInstr)) || X.ast_consts.ensure((n_consts + 1) * sizeof(fe))) return 1;
    std::vector<PolyBuf *> cols(polys);
    cols.push_back(nullptr);                                     // a program without operands still gets a table
    ColTable t;
    if (col_table(cols, nullptr, 0, s, &t)) return 1;
    CU(cudaMemcpyAsync(X.ast_code.p, code, n_code * sizeof(AstInstr), cudaMemcpyHostToDevice, s));
    if (h.up(P::ID, X.ast_consts.as<fe>(), consts, n_consts, s)) return 1;
    AstArgs A;
    A.polys = t.cols; A.code = X.ast_code.as<AstInstr>(); A.n_code = (uint32_t)n_code; A.consts = X.ast_consts.as<fe>();
    A.tw = nullptr; A.lin_base = fe_one<P>(); A.log_n = log_n; A.out = out->buf.as<fe>();
    if (has_linear) {
        if (get_twiddles_any(out->field, h.elem<P>(omega), log_n, s, &A.tw)) return 1;
        A.lin_base = h.elem<P>(lin_base);
    }
    LAUNCH(ast_eval_kernel<P>, blocks_for(n, 128), 128, 0, s, A);
    return 0;
}
extern "C" int h2_poly_eval_ast(uint64_t out, const uint64_t *polys, size_t n_polys, uint32_t log_n, const uint32_t *code, size_t n_code,
                                const void *consts, size_t n_consts, const void *omega, const void *lin_base, int repr) {
    CtxLock lk;
    if (require_ready()) return 1;
    if (log_n > 30) return fail("h2_poly_eval_ast: log_n > 30");
    if (n_code == 0 || n_code > (1u << 20)) return fail("h2_poly_eval_ast: empty or oversized program");
    PolyArgs g("h2_poly_eval_ast");
    std::vector<PolyBuf *> ps;
    PolyBuf *o = g.out(out, "out", (size_t)1 << log_n, "2^log_n");
    if (!o || g.in(polys, n_polys, "polys", (size_t)1 << log_n, "2^log_n", ps) || g.distinct()) return 1;   // operands are read at other rows
    const AstInstr *prog = reinterpret_cast<const AstInstr *>(code);
    int depth = 0;
    bool has_linear = false;
    for (size_t pc = 0; pc < n_code; pc++) {
        const AstInstr &in = prog[pc];
        switch (in.op) {
        case AST_POLY: if (in.arg >= n_polys) return fail("h2_poly_eval_ast: polynomial index out of range"); depth++; break;
        case AST_LINEAR: has_linear = true;   /* fall through */
        case AST_CONST: if (in.arg >= n_consts) return fail("h2_poly_eval_ast: constant index out of range"); depth++; break;
        case AST_ADD: case AST_MUL: if (depth < 2) return fail("h2_poly_eval_ast: operand stack underflow"); depth--; break;
        case AST_SCALE: if (in.arg >= n_consts) return fail("h2_poly_eval_ast: constant index out of range");   /* fall through */
        case AST_NEG: if (depth < 1) return fail("h2_poly_eval_ast: operand stack underflow"); break;
        default: return fail("h2_poly_eval_ast: unknown opcode");
        }
        if (depth > H2_AST_STACK) return fail("h2_poly_eval_ast: expression deeper than the operand stack (24)");
    }
    if (depth != 1) return fail("h2_poly_eval_ast: the program must leave exactly one value");
    const HostArgs h("h2_poly_eval_ast", repr);   // a LinearTerm needs omega and the coset generator
    if (h.check({{consts, "consts", n_consts != 0}, {omega, "omega", has_linear}, {lin_base, "lin_base", has_linear}})) return 1;
    return by_field(o->field, [&](auto p) { return ast_run<decltype(p)>(o, ps, log_n, prog, n_code, consts, n_consts, omega, lin_base, h, has_linear); });
}
// ff::BatchInvert on the first n elements of a resident polynomial, in place (zeros stay zero)
extern "C" int h2_poly_batch_invert(uint64_t poly, size_t n) {
    CtxLock lk;
    if (require_ready()) return 1;
    PolyArgs g("h2_poly_batch_invert");
    PolyBuf *a = g.out(poly, "poly", n, "n");
    if (!a) return 1;
    if (n == 0) return 0;
    cudaStream_t s = g_ctx.stream;
    const uint32_t nb = blocks_for((n + 15) / 16, 64);
    return by_field(a->field, [&](auto p) {
        LAUNCH(poly_batch_invert_kernel<decltype(p)>, nb, 64, 0, s, a->buf.as<fe>(), (uint64_t)n);
        return 0;
    });
}
// dst[0] = init, dst[i] = dst[i - 1] * src[i - 1] for i < n: the running product of plonk/permutation/prover.rs:150-156
template <class P> static int grand_product_run(PolyBuf *d, PolyBuf *a, size_t n, const void *init, const HostArgs &h) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    GpTree T;
    if (const char *e = gp_scan_plan(n, 1, false, &T)) return fail(std::string(h.who) + ": " + e);
    const uint64_t *m = T.m, *off = T.off;
    const size_t L = T.L;
    if (X.po_lvl.ensure(T.total * sizeof(fe)) || X.po_q.ensure(T.total * sizeof(fe))) return 1;
    fe *lvl = X.po_lvl.as<fe>(), *ex = X.po_q.as<fe>();
    const fe *src = a->buf.as<fe>();
    const fe in0 = h.elem<P>(init);
    for (size_t l = 0; l < L; l++)
        LAUNCH(poly_product_up_kernel<P>, blocks_for(m[l + 1], 128), 128, 0, s, l == 0 ? src : (const fe *)(lvl + off[l]), m[l], lvl + off[l + 1], m[l + 1]);
    for (size_t l = L + 1; l-- > 0;) {
        const uint64_t chunks = (m[l] + H2_POLY_CHUNK - 1) / H2_POLY_CHUNK;
        LAUNCH(poly_product_down_kernel<P>, blocks_for(chunks, 128), 128, 0, s, l == 0 ? src : (const fe *)(lvl + off[l]), m[l],
               l == L ? (const fe *)nullptr : (const fe *)(ex + off[l + 1]), in0, l == 0 ? d->buf.as<fe>() : ex + off[l], chunks);
    }
    return 0;
}
extern "C" int h2_poly_running_product(uint64_t dst, uint64_t src, size_t n, const void *init, int repr) {
    CtxLock lk;
    const HostArgs h("h2_poly_running_product", repr);
    if (require_ready() || h.check({{init, "init", n != 0}})) return 1;
    PolyArgs g("h2_poly_running_product");
    PolyBuf *d, *a;
    if (!(d = g.out(dst, "dst", n, "n")) || !(a = g.in(src, "src", n, "n")) || g.distinct()) return 1;
    if (n == 0) return 0;
    return by_field(a->field, [&](auto p) { return grand_product_run<decltype(p)>(d, a, n, init, h); });
}
// divide_by_vanishing_poly on a resident extended-domain polynomial; t_evals: t_len = 2^(ext_k - k) host elements
extern "C" int h2_poly_divide_by_vanishing(uint64_t poly, uint32_t ext_k, const void *t_evals, uint32_t t_len, int repr) {
    CtxLock lk;
    const HostArgs h("h2_poly_divide_by_vanishing", repr);
    if (require_ready() || h.check({{t_evals, "t_evals"}})) return 1;
    if (ext_k > 30) return fail("h2_poly_divide_by_vanishing: ext_k > 30");
    PolyArgs g("h2_poly_divide_by_vanishing");
    PolyBuf *a = g.out(poly, "poly", (size_t)1 << ext_k, "2^ext_k");
    if (!a) return 1;
    if (t_len == 0 || (t_len & (t_len - 1)) || t_len > (1u << ext_k)) return fail("h2_poly_divide_by_vanishing: t_len must be a power of two <= 2^ext_k");
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (X.po_pts.ensure((size_t)t_len * sizeof(fe))) return 1;
    if (h.up(a->field, X.po_pts.as<fe>(), t_evals, t_len, s)) return 1;
    const uint64_t n = 1ull << ext_k;
    return by_field(a->field, [&](auto p) {
        LAUNCH(poly_vanish_div_kernel<decltype(p)>, blocks_for(n, 256), 256, 0, s, a->buf.as<fe>(), n, (const fe *)X.po_pts.as<fe>(), t_len - 1);
        return 0;
    });
}
extern "C" int h2_poly_eval(const uint64_t *polys, size_t batch, size_t n, const void *points, int repr, void *out) {
    const HostArgs h("h2_poly_eval", repr);
    if (h.check({{points, "points", batch != 0 && n != 0}, {out, "out", batch != 0}})) return 1;
    if (n == 0) { memset(out, 0, batch * 32); return 0; }            // the empty sum (fold over nothing, arithmetic.rs:300-302)
    return polyops_dispatch(0, polys, nullptr, batch, n, points, h, out);
}
extern "C" int h2_poly_inner_product(const uint64_t *a, const uint64_t *b, size_t batch, size_t n, int repr, void *out) {
    const HostArgs h("h2_poly_inner_product", repr);
    if (h.check({{out, "out", batch != 0}})) return 1;
    if (n == 0) { memset(out, 0, batch * 32); return 0; }
    return polyops_dispatch(1, a, b, batch, n, nullptr, h, out);
}
extern "C" int h2_poly_kate_division(const uint64_t *dst, const uint64_t *src, size_t batch, size_t n, const void *points, int repr) {
    const HostArgs h("h2_poly_kate_division", repr);
    if (h.check({{points, "points", batch != 0 && n > 1}})) return 1;
    if (n == 0) return fail("h2_poly_kate_division: empty polynomial (the reference underflows a.len() - 1, arithmetic.rs:329)");
    if (n == 1) return 0;                                             // quotient of a constant: no coefficients
    return polyops_dispatch(2, src, dst, batch, n, points, h, nullptr);
}



// ------------------------------------------------------------------------------------------------
// the lookup argument's permuted columns (lookup.cuh)
// ------------------------------------------------------------------------------------------------
static int lk_scan(uint32_t *d, uint64_t n, cudaStream_t s) {     // exclusive scan in place (kernels of msm.cuh)
    const uint64_t per_block = (uint64_t)H2_SCAN_BLOCK * H2_SCAN_ITEMS;
    const uint32_t nb = (uint32_t)((n + per_block - 1) / per_block);
    if (g_ctx.scan_blocks.ensure((size_t)nb * 4 + 16)) return 1;
    uint32_t *bs = g_ctx.scan_blocks.as<uint32_t>();
    LAUNCH(scan_block_sums_kernel, nb, H2_SCAN_BLOCK, 0, s, d, n, bs, (const uint32_t *)nullptr);
    LAUNCH(scan_single_block_kernel, 1, H2_SCAN_BLOCK, 0, s, bs, nb, (const uint32_t *)nullptr);
    LAUNCH(scan_apply_kernel, nb, H2_SCAN_BLOCK, 0, s, d, n, bs, (const uint32_t *)nullptr);
    return 0;
}
// ascending bitonic sort of `count` arrays of N = 2^m canonical keys each, one per grid.y
template <class P> static int lk_sort(fe *keys, uint64_t N, uint32_t count, cudaStream_t s) {
    const uint64_t BL = N < (1ull << H2_LK_BLOCK_LOG) ? N : (1ull << H2_LK_BLOCK_LOG);
    const uint32_t smem = (uint32_t)(BL * sizeof(fe)), thr = (uint32_t)(BL / 2 < 512 ? (BL / 2 ? BL / 2 : 1) : 512);
    const dim3 blocks((uint32_t)(N / BL), count), stage(blocks_for(N / 2, 256), count);
    LAUNCH(lk_bitonic_block_kernel, blocks, thr, smem, s, keys, N, (uint64_t)2, 1u);
    for (uint64_t size = 2 * BL; size <= N; size <<= 1) {
        for (uint64_t stride = size / 2; stride >= BL; stride >>= 1) {
            LAUNCH(lk_bitonic_global_kernel<P>, stage, 256, 0, s, keys, N, size, stride);
        }
        LAUNCH(lk_bitonic_block_kernel, blocks, thr, smem, s, keys, N, size, 0u);
    }
    return 0;
}
// The permuted columns of `count` lookups of u usable rows (lookup.cuh), and with `blinding` (count x 2 rows values) the
// blinding rows [u, u + rows) of every output.  Scratch from the lane's pools: lk_keys and lk_u32 as lk_plan lays them out,
// col_tab 32 bytes of pointers + 64 rows bytes of blinding values per lookup, 4 bytes per 8192 scanned words.
// `h`: the encoding of the blinding values (nullptr without them).  One synchronisation; *bad = the lowest lookup with an input value
// its table lacks, H2_LK_NONE when none -- and then every output is as it was (the one writing kernel runs after the miss is known and
// checks for it first).
template <class P>
static int lookup_permuted_run(const std::vector<PolyBuf *> &out_in, const std::vector<PolyBuf *> &out_tab, const std::vector<PolyBuf *> &in,
                               const std::vector<PolyBuf *> &tab, uint64_t u, uint64_t rows, const void *blinding, const HostArgs *h, uint32_t *bad) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint32_t count = (uint32_t)in.size();
    const LkPlan plan = lk_plan(u, count);
    const uint64_t N = plan.N, w = plan.w, nblind = blinding ? (uint64_t)count * 2 * rows : 0;
    std::vector<PolyBuf *> cols(in);                             // LkCols: in, tab, out_in, out_tab
    for (auto *v : {&tab, &out_in, &out_tab}) cols.insert(cols.end(), v->begin(), v->end());
    if (X.lk_keys.ensure(plan.keys_end * sizeof(fe)) || X.lk_u32.ensure(plan.u32_end * sizeof(uint32_t))) return 1;
    fe *keys = X.lk_keys.as<fe>() + plan.keys;
    uint32_t *u32 = X.lk_u32.as<uint32_t>(), *sc = u32 + plan.sc, *left = u32 + plan.left, *err = u32 + plan.err;
    ColTable t;
    if (col_table(cols, blinding, nblind * sizeof(fe), s, &t)) return 1;
    LkCols c;
    c.in = t.cols;
    c.tab = c.in + count;
    c.out_in = t.cols + 2 * count;
    c.out_tab = c.out_in + count;
    c.blind = t.data;
    if (nblind && h->to_mont(P::ID, t.data, nblind, s)) return 1;
    CU(cudaMemsetAsync(sc, 0, w * count * sizeof(uint32_t), s));
    CU(cudaMemsetAsync(err, 0xFF, sizeof(uint32_t), s));
    LAUNCH(lk_load_kernel<P>, dim3(blocks_for(N, 256), count), 256, 0, s, c, u, keys, N);
    if (lk_sort<P>(keys, N, count, s)) return 1;
    LAUNCH(lk_rank_kernel<P>, dim3(blocks_for(u, 128), count), 128, 0, s, c, (const fe *)keys, N, u, sc, err);
    LAUNCH(lk_unconsumed_kernel, dim3(blocks_for(w, 256), count), 256, 0, s, sc, u, count);
    if (lk_scan(sc, 2 * w * count, s)) return 1;
    LAUNCH(lk_leftover_kernel, dim3(blocks_for(u, 256), count), 256, 0, s, (const uint32_t *)sc, u, count, left);
    LAUNCH(lk_fill_kernel<P>, dim3(blocks_for(u + (nblind ? rows : 0), 256), count), 256, 0, s, c, (const fe *)keys, N, u, rows, (const uint32_t *)sc, count,
           (const uint32_t *)left, (const uint32_t *)err);
    CU(cudaMemcpyAsync(bad, err, sizeof *bad, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return 0;
}
static const char *lk_miss = "an input value does not occur in the table (Error::ConstraintSystemFailure, plonk/lookup/prover.rs:605-608)";
extern "C" int h2_poly_lookup_permute(uint64_t input, uint64_t table, size_t usable_rows, uint64_t out_input, uint64_t out_table) {
    static const char *who = "h2_poly_lookup_permute";
    CtxLock lk;
    if (require_ready()) return 1;
    PolyArgs g(who);
    PolyBuf *oi, *ot, *i, *t;
    if (!(oi = g.out(out_input, "out_input", usable_rows, "usable_rows")) || !(ot = g.out(out_table, "out_table", usable_rows, "usable_rows")) ||
        !(i = g.in(input, "input", usable_rows, "usable_rows")) || !(t = g.in(table, "table", usable_rows, "usable_rows")) || g.distinct())
        return 1;
    if (usable_rows >= (1ull << 31)) return fail("h2_poly_lookup_permute: usable_rows >= 2^31");
    if (usable_rows == 0) return 0;
    uint32_t bad = H2_LK_NONE;
    if (by_field(oi->field, [&](auto p) { return lookup_permuted_run<decltype(p)>({oi}, {ot}, {i}, {t}, usable_rows, 0, nullptr, nullptr, &bad); }))
        return 1;
    if (bad != H2_LK_NONE) return fail(std::string(who) + ": " + lk_miss);
    return 0;
}
extern "C" int h2_poly_lookup_permuted(const uint64_t *out_inputs, const uint64_t *out_tables, size_t count, const uint64_t *inputs, const uint64_t *tables,
                                       uint32_t k, const void *blinding, uint32_t blinding_factors, int repr) {
    static const char *who = "h2_poly_lookup_permuted";
    CtxLock lk;
    const HostArgs h(who, repr);
    if (require_ready() || h.check({{blinding, "blinding", count != 0}})) return 1;
    if (k > 30) return fail(std::string(who) + ": k > 30");
    if ((uint64_t)blinding_factors + 1 >= (1ull << k)) return fail(std::string(who) + ": blinding_factors + 1 >= n");
    if (count == 0) return 0;
    if (!out_inputs || !out_tables || !inputs || !tables) return fail(std::string(who) + ": null argument");
    if (count > 65535) return fail(std::string(who) + ": more than 65535 lookups");
    const uint64_t n = 1ull << k, rows = (uint64_t)blinding_factors + 1;
    PolyArgs g(who);
    std::vector<PolyBuf *> oi, ot, i, t;
    if (g.out(out_inputs, count, "out_inputs", n, "2^k", oi) || g.out(out_tables, count, "out_tables", n, "2^k", ot) ||
        g.in(inputs, count, "inputs", n, "2^k", i) || g.in(tables, count, "tables", n, "2^k", t) || g.distinct())
        return 1;
    uint32_t bad = H2_LK_NONE;
    if (by_field(oi[0]->field, [&](auto p) { return lookup_permuted_run<decltype(p)>(oi, ot, i, t, n - rows, rows, blinding, &h, &bad); })) return 1;
    if (bad != H2_LK_NONE) return fail(std::string(who) + ": lookup " + std::to_string(bad) + ": " + lk_miss);
    return 0;
}


// ------------------------------------------------------------------------------------------------
// the verifier's MSM: g_scalars resident (verifier.cuh)
// ------------------------------------------------------------------------------------------------
// dst[i] (+)= init * prod_{j : bit j of i} u[k - 1 - j], i < 2^k: compute_s (poly/commitment/verifier.rs:156-171); with
// `accumulate` the add_to_g_scalars of Guard::use_challenges (:36-41, msm.rs:104-113) in the same pass
template <class P> static int compute_s_run(PolyBuf *d, const void *u, uint32_t k, const void *init, int accumulate, const HostArgs &h) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (X.po_pts.ensure((size_t)k * sizeof(fe))) return 1;
    fe *du = X.po_pts.as<fe>();
    if (h.up(P::ID, du, u, k, s)) return 1;
    const uint64_t groups = 1ull << (k - (k < 2 ? k : 2));
    LAUNCH(verifier_compute_s_kernel<P>, blocks_for(groups, 128), 128, 0, s, d->buf.as<fe>(), (const fe *)du, k, h.elem<P>(init), accumulate);
    return 0;
}
extern "C" int h2_poly_compute_s(uint64_t dst, const void *u, uint32_t k, const void *init, int accumulate, int repr) {
    CtxLock lk;
    const HostArgs h("h2_poly_compute_s", repr);
    if (require_ready() || h.check({{u, "u"}, {init, "init"}})) return 1;
    if (k == 0) return fail("h2_poly_compute_s: no challenges (assert!(!u.is_empty()), poly/commitment/verifier.rs:157)");
    if (k > 30) return fail("h2_poly_compute_s: k > 30");
    PolyArgs g("h2_poly_compute_s");
    PolyBuf *d = g.out(dst, "dst", (size_t)1 << k, "2^k");
    if (!d) return 1;
    return by_field(d->field, [&](auto p) { return compute_s_run<decltype(p)>(d, u, k, init, accumulate, h); });
}
// dst[i] = a * dst[i] + b * src[i], i < n (src == 0: dst[i] *= a): MSM::scale and the g_scalars part of MSM::add_msm
// (poly/commitment/msm.rs:126-139, :37-62); BatchVerifier's accumulate_msm (plonk/verifier/batch.rs:83-93) is one call
extern "C" int h2_poly_scale_add(uint64_t dst, const void *a, uint64_t src, const void *b, size_t n, int repr) {
    CtxLock lk;
    const HostArgs h("h2_poly_scale_add", repr);
    if (require_ready() || h.check({{a, "a"}, {b, "b", src != 0}})) return 1;
    PolyArgs g("h2_poly_scale_add");
    PolyBuf *d = g.out(dst, "dst", n, "n"), *x = nullptr;
    if (!d || (src && !(x = g.in(src, "src", n, "n"))) || g.distinct()) return 1;
    if (n == 0) return 0;
    cudaStream_t s = g_ctx.stream;
    const fe *sp = x ? x->buf.as<fe>() : nullptr;
    return by_field(d->field, [&](auto p) {
        using P = decltype(p);
        LAUNCH(verifier_scale_add_kernel<P>, blocks_for(n, 256), 256, 0, s, d->buf.as<fe>(), sp, h.elem<P>(a), x ? h.elem<P>(b) : fe_zero(), (uint64_t)n);
        return 0;
    });
}


// ------------------------------------------------------------------------------------------------
// the permutation argument's sigma polynomials (keygen.cuh)
// ------------------------------------------------------------------------------------------------
// The mapping goes up in pieces of at most this many (column, row) pairs, so the scratch it needs stays at 32 MB whatever
// the circuit's size; every piece is ordered on the context's stream behind the kernel that read the previous one.
#define H2_KEYGEN_CHUNK (1ull << 22)
// The launches both entry points share: the power tables, then one sigma launch per (column, piece) of the mapping, then
// the error word back.  sigma_finish synchronises.
template <class P>
static int sigma_tables(uint32_t k, uint64_t cols, const void *omega, const void *delta, const HostArgs &h, fe **tab, uint32_t **err) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint64_t tlen = KeygenOps<P>::table_len(k, (uint32_t)cols);
    if (X.kg_tab.ensure(tlen * sizeof(fe) + 16)) return 1;
    *tab = X.kg_tab.as<fe>();
    *err = reinterpret_cast<uint32_t *>(*tab + tlen);
    CU(cudaMemsetAsync(*err, 0, sizeof(uint32_t), s));
    LAUNCH(keygen_tables_kernel<P>, blocks_for(tlen, 128), 128, 0, s, *tab, h.elem<P>(omega), h.elem<P>(delta), k, (uint32_t)cols);
    return 0;
}
template <class P>
static int sigma_launch(PolyBuf *d, uint64_t j0, const uint2 *map, uint64_t len, uint32_t k, uint64_t cols, const fe *tab, uint32_t *err) {
    LAUNCH(keygen_sigma_kernel<P>, blocks_for(len, 256), 256, 0, g_ctx.stream, d->buf.as<fe>() + j0, map, tab, k, (uint32_t)cols, len, err);
    return 0;
}
static int sigma_finish(uint32_t *err, const char *who) {
    cudaStream_t s = g_ctx.stream;
    uint32_t h_err = 0;
    CU(cudaMemcpyAsync(&h_err, err, sizeof h_err, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (h_err) return fail(std::string(who) + ": a mapping entry is outside the permutation's columns or the domain's rows");
    return 0;
}
template <class P>
static int permutation_sigma_run(const std::vector<PolyBuf *> &dst, uint32_t k, const uint32_t *mapping, const void *omega, const void *delta,
                                 const HostArgs &h) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint64_t n = 1ull << k, cols = dst.size();
    const uint64_t piece = n < H2_KEYGEN_CHUNK ? n : H2_KEYGEN_CHUNK;
    fe *tab;
    uint32_t *err;
    if (X.kg_map.ensure(piece * sizeof(uint2)) || sigma_tables<P>(k, cols, omega, delta, h, &tab, &err)) return 1;
    uint2 *map = X.kg_map.as<uint2>();
    for (uint64_t i = 0; i < cols; i++)
        for (uint64_t j0 = 0; j0 < n; j0 += piece) {
            const uint64_t len = n - j0 < piece ? n - j0 : piece;
            if (upload_async(map, mapping + 2 * (i * n + j0), len * sizeof(uint2), s)) return 1;
            if (sigma_launch<P>(dst[i], j0, map, len, k, cols, tab, err)) return 1;
        }
    return sigma_finish(err, "h2_poly_permutation_sigma");
}
extern "C" int h2_poly_permutation_sigma(const uint64_t *dst, size_t cols, uint32_t k, const uint32_t *mapping, const void *omega, const void *delta,
                                         int repr) {
    CtxLock lk;
    const HostArgs h("h2_poly_permutation_sigma", repr);
    if (require_ready() || h.check({{omega, "omega", cols != 0}, {delta, "delta", cols != 0}})) return 1;
    if (k > 30) return fail("h2_poly_permutation_sigma: k > 30");
    if (cols == 0) return 0;
    if (cols >= (1ull << 32)) return fail("h2_poly_permutation_sigma: cols >= 2^32");
    if (!dst || !mapping) return fail("h2_poly_permutation_sigma: null argument");
    PolyArgs g("h2_poly_permutation_sigma");
    std::vector<PolyBuf *> d;
    if (g.out(dst, cols, "dst", (size_t)1 << k, "2^k", d) || g.distinct()) return 1;
    return by_field(d[0]->field, [&](auto p) { return permutation_sigma_run<decltype(p)>(d, k, mapping, omega, delta, h); });
}


// ------------------------------------------------------------------------------------------------
// the permutation argument's copy cycles from the copy constraints (assembly.cuh), then sigma (keygen.cuh)
// ------------------------------------------------------------------------------------------------
static int as_read_u32(uint32_t *h, const uint32_t *d, cudaStream_t s) {     // one device word back, synchronously
    CU(cudaMemcpyAsync(h, d, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return 0;
}
// The copy-cycle mapping of m copies (4 uint32 each, synthesis order) over cols * 2^k cells into X.kg_map as (column,
// row) pairs; *bad = 2 i (column) / 2 i + 1 (row) of the first bad copy i, or ~0.  Scratch in the lane's pools: as_edge
// and as_slot as assembly.cuh lays them out, as_cell u32: comp N | best N.
static int assembly_run(uint32_t cols, uint32_t k, const uint32_t *copies, uint64_t m, unsigned long long *bad) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint64_t N = (uint64_t)cols << k;
    const AsEdgeLayout E = as_edge_layout(m);
    if (X.kg_map.ensure(N * sizeof(uint2)) || X.as_edge.ensure(E.end * sizeof(uint32_t))) return 1;
    uint2 *map = X.kg_map.as<uint2>();
    uint32_t *edge = X.as_edge.as<uint32_t>();
    unsigned long long *err = reinterpret_cast<unsigned long long *>(edge + E.err);
    uint32_t *changed = edge + E.changed, *cp = edge + E.copies, *ea = edge + E.ea, *eb = edge + E.eb, *flag = edge + E.flag;
    uint32_t *live[2] = {edge + E.live[0], edge + E.live[1]}, *ra = edge + E.ra, *rb = edge + E.rb, *keep = edge + E.keep, *fl = edge + E.fl;
    CU(cudaMemsetAsync(err, 0xFF, sizeof *err, s));
    if (m) {
        if (upload_async(cp, copies, m * 4 * sizeof(uint32_t), s)) return 1;
        LAUNCH(as_encode_kernel, blocks_for(m + 1, 256), 256, 0, s, (const uint32_t *)cp, (uint32_t)m, cols, k, ea, eb, flag, err);
    }
    CU(cudaMemcpyAsync(bad, err, sizeof *bad, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    if (*bad != ~0ull) return 0;
    LAUNCH(as_identity_kernel, blocks_for(N, 256), 256, 0, s, map, N, k);
    if (m == 0) return 0;
    // 2. the spanning forest, Borůvka rounds over the live copies
    uint32_t L = 0, q = 0;
    if (lk_scan(flag, m + 1, s) || as_read_u32(&L, flag + m, s)) return 1;
    LAUNCH(as_compact_kernel, blocks_for(m, 256), 256, 0, s, (const uint32_t *)flag, (uint32_t)m, (const uint32_t *)nullptr, live[0]);
    CU(cudaMemsetAsync(keep, 0, (m + 1) * sizeof(uint32_t), s));
    if (L) {
        if (X.as_cell.ensure(2 * N * sizeof(uint32_t))) return 1;
        uint32_t *comp = X.as_cell.as<uint32_t>(), *best = comp + N;
        LAUNCH(as_iota_kernel, blocks_for(N, 256), 256, 0, s, comp, N);
        const uint32_t limit = as_round_limit(N);
        for (uint32_t round = 0, cur = 0; L; round++, cur ^= 1) {
            if (round == limit) return fail("h2_poly_permutation_sigma_copies: internal error: the spanning forest needs more than log2(cells) rounds");
            const uint32_t *lv = live[cur];
            LAUNCH(as_roots_kernel, blocks_for(L, 256), 256, 0, s, lv, L, (const uint32_t *)ea, (const uint32_t *)eb, (const uint32_t *)comp, ra, rb, best);
            LAUNCH(as_best_kernel, blocks_for(L, 256), 256, 0, s, lv, L, (const uint32_t *)ra, (const uint32_t *)rb, best);
            LAUNCH(as_hook_kernel, blocks_for(L, 256), 256, 0, s, lv, L, (const uint32_t *)ra, (const uint32_t *)rb, (const uint32_t *)best, comp, keep);
            for (uint32_t h_changed = 1; h_changed;) {
                CU(cudaMemsetAsync(changed, 0, sizeof(uint32_t), s));
                LAUNCH(as_jump_kernel, blocks_for(N, 256), 256, 0, s, comp, N, changed);
                if (as_read_u32(&h_changed, changed, s)) return 1;
            }
            LAUNCH(as_split_kernel, blocks_for(L + 1, 256), 256, 0, s, lv, L, (const uint32_t *)ea, (const uint32_t *)eb, (const uint32_t *)comp, flag);
            if (lk_scan(flag, L + 1, s)) return 1;
            LAUNCH(as_compact_kernel, blocks_for(L, 256), 256, 0, s, (const uint32_t *)flag, L, lv, live[cur ^ 1]);
            if (as_read_u32(&L, flag + L, s)) return 1;
        }
    }
    if (lk_scan(keep, m + 1, s) || as_read_u32(&q, keep + m, s)) return 1;
    if (q == 0) return 0;
    LAUNCH(as_compact_kernel, blocks_for(m, 256), 256, 0, s, (const uint32_t *)keep, (uint32_t)m, (const uint32_t *)nullptr, fl);
    // 3. slots, stably sorted by cell
    const uint64_t S = 2ull * q;
    if (S >= (1ull << 32)) return fail("h2_poly_permutation_sigma_copies: the spanning forest has 2^31 copies or more");
    const AsSlotLayout Q = as_slot_layout(S);
    const uint64_t ntiles = Q.ntiles;
    if (X.as_slot.ensure(Q.end * sizeof(uint32_t))) return 1;
    uint32_t *slot = X.as_slot.as<uint32_t>(), *scell = slot + Q.scell, *order[2] = {slot + Q.order[0], slot + Q.order[1]};
    uint32_t *nxt[2] = {slot + Q.nxt[0], slot + Q.nxt[1]}, *counts = slot + Q.counts;
    LAUNCH(as_slots_kernel, blocks_for(S, 256), 256, 0, s, (const uint32_t *)fl, S, (const uint32_t *)ea, (const uint32_t *)eb, scell, order[0]);
    uint32_t o = 0;
    for (uint32_t shift = 0; shift == 0 || ((N - 1) >> shift); shift += H2_AS_DIGIT_BITS, o ^= 1) {
        LAUNCH(as_radix_hist_kernel, (uint32_t)ntiles, H2_AS_TILE, 0, s, (const uint32_t *)order[o], S, (const uint32_t *)scell, shift, ntiles, counts);
        if (lk_scan(counts, H2_AS_TILE * ntiles + 1, s)) return 1;
        LAUNCH(as_radix_scatter_kernel, (uint32_t)ntiles, H2_AS_TILE, 0, s, (const uint32_t *)order[o], S, (const uint32_t *)scell, shift,
               (const uint32_t *)counts, ntiles, order[o ^ 1]);
    }
    // 4. successor and pointer jumping: a walk has at most |F| steps < 2^rounds
    LAUNCH(as_succ_kernel, blocks_for(S, 256), 256, 0, s, (const uint32_t *)order[o], S, (const uint32_t *)scell, nxt[0]);
    uint32_t t = 0;
    for (uint64_t len = 1; len <= S; len <<= 1, t ^= 1)
        LAUNCH(as_jump_slots_kernel, blocks_for(S, 256), 256, 0, s, (const uint32_t *)nxt[t], nxt[t ^ 1], S);
    LAUNCH(as_final_kernel, blocks_for(S, 256), 256, 0, s, (const uint32_t *)order[o], S, (const uint32_t *)scell, (const uint32_t *)nxt[t], k, map);
    return 0;
}
template <class P>
static int permutation_sigma_copies_run(const std::vector<PolyBuf *> &dst, uint32_t k, const uint32_t *copies, uint64_t m, const void *omega,
                                        const void *delta, const HostArgs &h) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint64_t n = 1ull << k, cols = dst.size();
    unsigned long long bad = ~0ull;
    if (assembly_run((uint32_t)cols, k, copies, m, &bad)) return 1;
    if (bad != ~0ull) {
        return fail("h2_poly_permutation_sigma_copies: copy " + std::to_string(bad >> 1) +
                    ((bad & 1) ? ": a row is outside the domain (Error::BoundsFailure)" : ": a column is outside the permutation (Error::ColumnNotInPermutation)"));
    }
    fe *tab;
    uint32_t *err;
    if (sigma_tables<P>(k, cols, omega, delta, h, &tab, &err)) return 1;
    const uint2 *map = X.kg_map.as<uint2>();
    for (uint64_t i = 0; i < cols; i++)
        if (sigma_launch<P>(dst[i], 0, map + i * n, n, k, cols, tab, err)) return 1;
    return sigma_finish(err, "h2_poly_permutation_sigma_copies");
}
extern "C" int h2_poly_permutation_sigma_copies(const uint64_t *dst, size_t cols, uint32_t k, const uint32_t *copies, size_t m, const void *omega,
                                                const void *delta, int repr) {
    CtxLock lk;
    const HostArgs h("h2_poly_permutation_sigma_copies", repr);
    if (require_ready() || h.check({{omega, "omega", cols != 0}, {delta, "delta", cols != 0}})) return 1;
    if (k > 30) return fail("h2_poly_permutation_sigma_copies: k > 30");
    if (cols == 0) return 0;
    if (cols >= (1ull << 32)) return fail("h2_poly_permutation_sigma_copies: cols >= 2^32");
    if (!dst || (m && !copies)) return fail("h2_poly_permutation_sigma_copies: null argument");
    if (((uint64_t)cols << k) >= (1ull << 32)) return fail("h2_poly_permutation_sigma_copies: cols * 2^k >= 2^32 cells");
    if ((uint64_t)m >= (1ull << 32)) return fail("h2_poly_permutation_sigma_copies: m >= 2^32 copies");
    PolyArgs g("h2_poly_permutation_sigma_copies");
    std::vector<PolyBuf *> d;
    if (g.out(dst, cols, "dst", (size_t)1 << k, "2^k", d) || g.distinct()) return 1;
    return by_field(d[0]->field, [&](auto p) { return permutation_sigma_copies_run<decltype(p)>(d, k, copies, m, omega, delta, h); });
}


// ------------------------------------------------------------------------------------------------
// the prover's random polynomials: ChaCha20Rng draws of Field::random (chacha.cuh)
// ------------------------------------------------------------------------------------------------
extern "C" int h2_poly_random(const uint64_t *polys, size_t count, const size_t *lens, const void *seed32, uint64_t stream, uint64_t block,
                              uint32_t word) {
    static const char *who = "h2_poly_random";
    CtxLock lk;
    if (require_ready()) return 1;
    if (count == 0) return fail(std::string(who) + ": count == 0");
    if (!polys || !lens) return fail(std::string(who) + ": null argument");
    if (!seed32) return fail(std::string(who) + ": null seed32");
    if (word >= 16) return fail(std::string(who) + ": word >= 16");
    PolyArgs g(who);
    std::vector<PolyBuf *> ps;
    if (g.out(polys, count, "polys", lens, "lens", ps) || g.distinct()) return 1;
    // draw j of the call reads blocks block + j and, with word != 0, block + j + 1: the last one must not pass 2^64 - 1
    std::vector<RandCol> cols(count);
    uint64_t total = 0, longest = 0;
    for (size_t i = 0; i < count; i++) {            // each lens[i] fits its polynomial, so the sum cannot wrap
        cols[i] = {total, (uint64_t)lens[i]};
        total += lens[i];
        longest = std::max<uint64_t>(longest, lens[i]);
    }
    if (total == 0) return 0;
    if (total - 1 + (word != 0) > ~0ull - block) return fail(std::string(who) + ": the draws run past keystream block 2^64 - 1");
    ChaChaKey key;
    memcpy(key.k, seed32, sizeof key.k);
    cudaStream_t s = g_ctx.stream;
    ColTable t;
    if (col_table(ps, cols.data(), count * sizeof(RandCol), s, &t)) return 1;
    return by_field(ps[0]->field, [&](auto p) {
        using P = decltype(p);
        for (size_t c0 = 0; c0 < count; c0 += 65535) {   // grid.y limit
            const uint32_t n = (uint32_t)std::min<size_t>(count - c0, 65535);
            LAUNCH(chacha_random_kernel<P>, dim3(blocks_for(longest, 256), n), 256, 0, s, t.cols, reinterpret_cast<const RandCol *>(t.data), (uint32_t)c0,
                   key, stream, block, word);
        }
        return 0;
    });
}


// ------------------------------------------------------------------------------------------------
// the permutation and lookup arguments' product columns, every column of every proof in one call (grandproduct.cuh)
// ------------------------------------------------------------------------------------------------
// `ins`: the permutation's proofs x cols column pointers then its cols sigma pointers, or 4 pointers per lookup column.
// Scratch: gp_val [count][n] (den, den^-1, mv), po_lvl / po_q the tree's levels and exclusive products, col_tab one upload of
// the pointer arrays (z, then ins) and the blinding values, gp_aux the power tables and the carries.
template <class P>
static int product_run(bool perm, const std::vector<PolyBuf *> &z, const std::vector<PolyBuf *> &ins, uint32_t ncols, uint32_t chunk_len,
                       uint32_t sets, uint32_t k, const void *beta, const void *gamma, const void *omega, const void *delta, const void *blinding,
                       uint32_t bf, const HostArgs &h) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const uint64_t n = 1ull << k, count = z.size();
    GpTree G;
    if (const char *e = gp_scan_plan(n, count, true, &G)) return fail(std::string(h.who) + ": " + e);
    const uint64_t tlen = perm ? KeygenOps<P>::table_len(k, ncols) : 0, nblind = count * bf;
    std::vector<PolyBuf *> cols(z);
    cols.insert(cols.end(), ins.begin(), ins.end());
    if (X.gp_val.ensure(count * n * sizeof(fe)) || X.po_lvl.ensure(G.total * sizeof(fe)) || X.po_q.ensure(G.total * sizeof(fe)) ||
        X.gp_aux.ensure((tlen + count) * sizeof(fe)))
        return 1;
    fe *val = X.gp_val.as<fe>(), *lvl = X.po_lvl.as<fe>(), *ex = X.po_q.as<fe>(), *tab = X.gp_aux.as<fe>(), *init = tab + tlen;
    ColTable t;
    if (col_table(cols, blinding, nblind * sizeof(fe), s, &t) || h.to_mont(P::ID, t.data, nblind, s)) return 1;
    fe *const *zp = t.cols;
    const fe *const *ip = t.cols + count;
    const fe b_m = h.elem<P>(beta), g_m = h.elem<P>(gamma);
    if (perm) {
        LAUNCH(keygen_tables_kernel<P>, blocks_for(tlen, 128), 128, 0, s, tab, h.elem<P>(omega), h.elem<P>(delta), k, ncols);
        LAUNCH(gp_perm_factors_kernel<P>, dim3(blocks_for(n, 128), (uint32_t)count), 128, 0, s, ip, ip + (count / sets) * ncols, ncols, chunk_len, sets,
               (const fe *)tab, k, b_m, g_m, val, zp);
    } else {
        LAUNCH(gp_lookup_factors_kernel<P>, dim3(blocks_for(n, 256), (uint32_t)count), 256, 0, s, ip, n, b_m, g_m, val, zp);
    }
    LAUNCH(poly_batch_invert_kernel<P>, blocks_for((count * n + 15) / 16, 64), 64, 0, s, val, count * n);
    LAUNCH(gp_mv_up_kernel<P>, dim3(blocks_for(G.m[1], 128), (uint32_t)count), 128, 0, s, (const fe *const *)zp, val, n, lvl, G.m[1]);
    for (uint32_t l = 1; l < G.L; l++)
        LAUNCH(gp_up_kernel<P>, dim3(blocks_for(G.m[l + 1], 128), (uint32_t)count), 128, 0, s, (const fe *)(lvl + G.off[l]), G.m[l], lvl + G.off[l + 1], G.m[l + 1]);
    LAUNCH(gp_carry_kernel<P>, blocks_for(count / sets, 64), 64, 0, s, (const fe *)val, (const fe *)lvl, (const GpLevels &)G, n - bf - 1, sets, init, (uint32_t)(count / sets));
    for (uint32_t l = G.L + 1; l-- > 0;) {
        const uint64_t chunks = (G.m[l] + H2_POLY_CHUNK - 1) / H2_POLY_CHUNK;
        LAUNCH(gp_down_kernel<P>, dim3(blocks_for(chunks, 128), (uint32_t)count), 128, 0, s, l == 0 ? (const fe *)val : (const fe *)(lvl + G.off[l]), G.m[l],
               l == G.L ? (const fe *)nullptr : (const fe *)(ex + G.off[l + 1]), (const fe *)init, l == 0 ? (fe *)nullptr : ex + G.off[l],
               l == 0 ? zp : (fe *const *)nullptr, chunks);
    }
    if (bf) LAUNCH(gp_blind_kernel<P>, blocks_for(nblind, 256), 256, 0, s, zp, n, bf, (const fe *)t.data, count);
    return 0;
}
static int product_scalars(const char *who, uint32_t k, uint32_t bf) {
    if (k > 30) return fail(std::string(who) + ": k > 30");
    if ((uint64_t)bf + 1 >= (1ull << k)) return fail(std::string(who) + ": blinding_factors + 1 >= n");
    return 0;
}
extern "C" int h2_poly_permutation_product(const uint64_t *z_out, size_t proofs, const uint64_t *columns, const uint64_t *sigmas, size_t cols,
                                           uint32_t chunk_len, uint32_t k, const void *beta, const void *gamma, const void *omega, const void *delta,
                                           const void *blinding, uint32_t blinding_factors, int repr) {
    static const char *who = "h2_poly_permutation_product";
    CtxLock lk;
    const HostArgs h(who, repr);
    const bool work = proofs != 0 && cols != 0;
    if (require_ready() || h.check({{beta, "beta", work}, {gamma, "gamma", work}, {omega, "omega", work}, {delta, "delta", work},
                                    {blinding, "blinding", work && blinding_factors != 0}}))
        return 1;
    if (product_scalars(who, k, blinding_factors)) return 1;
    if (chunk_len == 0) return fail(std::string(who) + ": chunk_len == 0");
    if (proofs == 0 || cols == 0) return 0;
    if (!z_out || !columns || !sigmas) return fail(std::string(who) + ": null argument");
    const uint64_t sets = (cols + chunk_len - 1) / chunk_len;
    if (cols >= (1ull << 20) || proofs >= (1ull << 16) || proofs * sets > 65535) return fail(std::string(who) + ": more than 65535 product columns");
    PolyArgs g(who);
    std::vector<PolyBuf *> z, ins, sig;
    if (g.out(z_out, proofs * sets, "z_out", 1ull << k, "2^k", z) || g.in(columns, proofs * cols, "columns", 1ull << k, "2^k", ins) ||
        g.in(sigmas, cols, "sigmas", 1ull << k, "2^k", sig) || g.distinct())
        return 1;
    ins.insert(ins.end(), sig.begin(), sig.end());
    return by_field(z[0]->field, [&](auto p) {
        return product_run<decltype(p)>(true, z, ins, (uint32_t)cols, chunk_len, (uint32_t)sets, k, beta, gamma, omega, delta, blinding, blinding_factors, h);
    });
}
extern "C" int h2_poly_lookup_product(const uint64_t *z_out, size_t count, const uint64_t *inputs, const uint64_t *tables, const uint64_t *permuted_inputs,
                                      const uint64_t *permuted_tables, uint32_t k, const void *beta, const void *gamma, const void *blinding,
                                      uint32_t blinding_factors, int repr) {
    static const char *who = "h2_poly_lookup_product";
    CtxLock lk;
    const HostArgs h(who, repr);
    const bool work = count != 0;
    if (require_ready() || h.check({{beta, "beta", work}, {gamma, "gamma", work}, {blinding, "blinding", work && blinding_factors != 0}})) return 1;
    if (product_scalars(who, k, blinding_factors)) return 1;
    if (count == 0) return 0;
    if (!z_out || !inputs || !tables || !permuted_inputs || !permuted_tables) return fail(std::string(who) + ": null argument");
    if (count > 65535) return fail(std::string(who) + ": more than 65535 product columns");
    const uint64_t n = 1ull << k;
    PolyArgs g(who);
    std::vector<PolyBuf *> z, in, tab, pin, ptab;
    if (g.out(z_out, count, "z_out", n, "2^k", z) || g.in(inputs, count, "inputs", n, "2^k", in) || g.in(tables, count, "tables", n, "2^k", tab) ||
        g.in(permuted_inputs, count, "permuted_inputs", n, "2^k", pin) || g.in(permuted_tables, count, "permuted_tables", n, "2^k", ptab) || g.distinct())
        return 1;
    std::vector<PolyBuf *> ins;                                  // gp_lookup_factors_kernel: 4 per column
    for (size_t b = 0; b < count; b++) ins.insert(ins.end(), {in[b], tab[b], pin[b], ptab[b]});
    return by_field(z[0]->field, [&](auto p) { return product_run<decltype(p)>(false, z, ins, 0, 1, 1, k, beta, gamma, nullptr, nullptr, blinding, blinding_factors, h); });
}
