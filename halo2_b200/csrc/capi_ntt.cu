// C ABI of the engine, part 3 of 5: the NTT pipeline (ntt.cuh), the domain transforms, device-resident polynomials.
#include "util_kernels.cuh"
#include "ntt.cuh"
#include "columns_io.cuh"

#include <algorithm>

// ------------------------------------------------------------------------------------------------
// NTT pipeline
// ------------------------------------------------------------------------------------------------
template <class P> static int get_twiddles(int field, const fe &omega_mont, uint32_t log_n, cudaStream_t s, const fe **out) {
    Context &X = g_ctx;
    fe canon = fe_from_mont<P>(omega_mont);
    for (auto *t : X.twiddles)
        if (t->field == field && t->log_n == log_n && memcmp(t->omega, canon.v, 32) == 0) {
            t->stamp = ++X.tw_stamp;
            *out = t->buf.as<fe>();
            return 0;
        }
    TwiddleEntry *e = nullptr;
    if (X.twiddles.size() >= 8) {   // evict least recently used
        size_t victim = 0;
        for (size_t i = 1; i < X.twiddles.size(); i++)
            if (X.twiddles[i]->stamp < X.twiddles[victim]->stamp) victim = i;
        e = X.twiddles[victim];
        X.twiddles.erase(X.twiddles.begin() + victim);
        CU(cudaStreamSynchronize(s));
    } else e = new TwiddleEntry();
    uint64_t half = log_n ? (1ull << (log_n - 1)) : 1;
    if (e->buf.ensure(half * sizeof(fe)) || X.pow2.ensure(64 * sizeof(fe))) { delete e; return 1; }
    e->field = field; e->log_n = log_n; memcpy(e->omega, canon.v, 32); e->stamp = ++X.tw_stamp;
    LAUNCH(twiddle_pow2_kernel<P>, 1, 32, 0, s, X.pow2.as<fe>(), omega_mont, log_n ? log_n : 1u);
    LAUNCH(twiddle_fill_kernel<P>, blocks_for((half + 31) / 32, 128), 128, 0, s, e->buf.as<fe>(), X.pow2.as<fe>(), half);
    X.twiddles.push_back(e);
    *out = e->buf.as<fe>();
    return 0;
}

struct NttScales {
    bool in_scale = false, out_scale = false;
    fe in_s[3], out_s[3];
    const fe *in_table = nullptr;   // device table: the first pass multiplies element j by in_table[j & in_mask] (NTT_IN_TABLE)
    uint32_t in_mask = 0;
    bool pieces = false;            // the last pass writes output p to out_cols[p >> piece_log] (NTT_OUT_PIECES; one column)
    uint32_t piece_log = 0;
};

// d_in: 2^in_log_n elements; d_out: min(out_len, 2^log_n) elements written.  d_out may alias d_in.
// With in_cols / out_cols (device tables of `count` pointers) the same transform runs on `count` columns, column c from
// in_cols[c] to out_cols[c] (d_in / d_out unused): every pass is one launch per group of columns (ntt.cuh: ntt_group), so a
// call whose columns fit in one group issues exactly the launches of one column.  out_cols[c] may alias in_cols[c] only.
template <class P>
static int ntt_run(int field, const fe *d_in, uint32_t in_log_n, fe *d_out, uint32_t log_n, const fe &omega_mont, const NttScales &sc,
                   uint64_t out_len, cudaStream_t s, uint64_t count = 1, const fe *const *in_cols = nullptr, fe *const *out_cols = nullptr) {
    Context &X = g_ctx;
    if (log_n > 30) return fail("ntt: log_n > 30 not supported");
    if (count == 0) return 0;
    uint64_t n = 1ull << log_n;
    const fe *tw = nullptr;
    if (get_twiddles<P>(field, omega_mont, log_n, s, &tw)) return 1;
    uint32_t sp[8], logc[8];
    int passes = ntt_plan(log_n, sp, logc);
    if (passes == 0) {   // n == 1: the network is empty; only the scalings apply
        sp[0] = 0; logc[0] = 0; passes = 1;
    }
    const uint64_t group = ntt_group(log_n, passes, count);
    if (passes > 1 && X.ntt_work.ensure(group * n * sizeof(fe))) return 1;
    static std::atomic<bool> smem_optin{false};   // per instantiation <P>: a single-CTA transform of 2^10 elements wants 64 KiB
    if (!smem_optin.load()) {
        CU(cudaFuncSetAttribute(ntt_pass_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        CU(cudaFuncSetAttribute(ntt_pass_tma_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        smem_optin = true;
    }
    for (uint64_t c0 = 0; c0 < count; c0 += group) {
        const uint32_t cols = (uint32_t)(count - c0 < group ? count - c0 : group);
        uint32_t s0 = 0;
        for (int i = 0; i < passes; i++) {
            NttPassArgs A;
            A.in = i == 0 ? d_in : X.ntt_work.as<fe>();
            A.out = i == passes - 1 ? d_out : X.ntt_work.as<fe>();
            if (i > 0) A.in_stride = n;
            if (i < passes - 1) A.out_stride = n;
            if (i == 0 && in_cols) A.in_cols = in_cols + c0;
            if (i == passes - 1 && out_cols) A.out_cols = out_cols + c0;
            A.tw = tw; A.log_n = log_n; A.s0 = s0; A.sp = sp[i]; A.logc = logc[i];
            A.flags = 0;
            if (i == 0) A.flags |= NTT_FIRST | (sc.in_scale ? NTT_IN_SCALE : 0u) | (sc.in_table ? NTT_IN_TABLE : 0u);
            if (i == passes - 1) A.flags |= NTT_LAST | (sc.out_scale ? NTT_OUT_SCALE : 0u) | (sc.pieces ? NTT_OUT_PIECES : 0u);
            A.in_table = sc.in_table; A.in_mask = sc.in_mask; A.piece_log = sc.piece_log;
            A.in_log_n = in_log_n; A.out_len = out_len;
            for (int k = 0; k < 3; k++) { A.in_scale[k] = sc.in_s[k]; A.out_scale[k] = sc.out_s[k]; }
            uint32_t tiles = (uint32_t)(n >> (sp[i] + logc[i]));
            uint32_t smem = ntt_smem_bytes(sp[i], logc[i]) + ntt_twc_bytes(sp[i], logc[i], i == passes - 1);
            prof_begin(PROF_NTT_PASS, s);
            if (X.ntt_tma && NttDense<P>::supported(A)) {
                // persistent CTAs (4 per SM by registers), double-buffered tiles on the bulk-copy engine
                int sms = 132;
                cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, X.device);
                // every CTA walks the same number of tiles (+-1): grid = tiles / ceil(tiles / resident CTAs)
                const uint32_t slots = (uint32_t)sms * 4u, per = (tiles + slots - 1) / slots;
                const uint32_t grid = (tiles + per - 1) / per;
                LAUNCH(ntt_pass_tma_kernel<P>, dim3(grid, cols), 128, ntt_tma_smem_bytes(sp[i], logc[i], i == passes - 1), s, A, tiles);
            } else
            LAUNCH(ntt_pass_kernel<P>, dim3(tiles, cols), 128, smem, s, A);
            prof_end(s);
            s0 += sp[i];
        }
    }
    return 0;
}

// Builds the in/out scale constants.  canon: the data enters and leaves in canonical form.
//   zeta_in  != null : multiply element j by zeta^(j mod 3)            (coeff_to_extended)
//   divisor  != null : multiply every output by divisor                (ifft)
//   zeta_out != null : multiply output p by [1, zeta^2, zeta][p mod 3] (extended_to_coeff)
template <class P>
static NttScales make_scales(bool canon, const fe *zeta_in, const fe *divisor, const fe *zeta_out) {
    NttScales sc;
    fe one = fe_one<P>();
    fe in_c[3] = {one, one, one}, out_c[3] = {one, one, one};
    bool in_needed = false, out_needed = false;
    if (zeta_in) { in_c[1] = *zeta_in; in_c[2] = fe_sqr<P>(*zeta_in); in_needed = true; }
    if (divisor) { for (int k = 0; k < 3; k++) out_c[k] = *divisor; out_needed = true; }
    if (zeta_out) { out_c[1] = fe_mul<P>(out_c[1], fe_sqr<P>(*zeta_out)); out_c[2] = fe_mul<P>(out_c[2], *zeta_out); out_needed = true; }
    if (canon) {
        // canonical -> Montgomery on the way in:  mont_mul(a, c R^2) = a c R
        for (int k = 0; k < 3; k++) in_c[k] = fe_mul<P>(in_c[k], fe_r2<P>());
        // Montgomery -> canonical on the way out: mont_mul(x R, c) = x c
        for (int k = 0; k < 3; k++) out_c[k] = fe_from_mont<P>(out_c[k]);
        in_needed = out_needed = true;
    }
    sc.in_scale = in_needed; sc.out_scale = out_needed;
    for (int k = 0; k < 3; k++) { sc.in_s[k] = in_c[k]; sc.out_s[k] = out_c[k]; }
    return sc;
}

// zeta / divisor: nullptr in the modes that have none (the entry points have checked the others)
template <class P> static NttScales host_scales(const HostArgs &h, bool canon, int mode, const void *zeta, const void *divisor) {
    const fe z = zeta ? h.elem<P>(zeta) : fe_zero(), d = divisor ? h.elem<P>(divisor) : fe_zero();
    return make_scales<P>(canon, mode == 2 ? &z : nullptr, (mode == 1 || mode == 3) ? &d : nullptr, mode == 3 ? &z : nullptr);
}
template <class P>
static int ntt_host(int field, int mode, const void *a_in, uint32_t in_log_n, uint32_t log_n, const void *omega, const void *zeta,
                    const void *divisor, size_t out_len, void *out, const HostArgs &h) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    uint64_t n = 1ull << log_n, n_in = 1ull << in_log_n;
    if (out_len > n) out_len = n;
    if (X.ntt_io.ensure(n_in * sizeof(fe)) || X.ntt_out.ensure(n * sizeof(fe))) return 1;
    const NttScales sc = host_scales<P>(h, h.canon(), mode, zeta, divisor);
    if (upload_async(X.ntt_io.p, a_in, n_in * sizeof(fe), s)) return 1;
    if (ntt_run<P>(field, X.ntt_io.as<fe>(), in_log_n, X.ntt_out.as<fe>(), log_n, h.elem<P>(omega), sc, out_len, s)) return 1;
    return download_sync(out, X.ntt_out.p, out_len * sizeof(fe), s);
}
static int ntt_host_dispatch(int field, int mode, const void *a_in, uint32_t in_log_n, uint32_t log_n, const void *omega, const void *zeta,
                             const void *divisor, size_t out_len, void *out, const HostArgs &h, std::initializer_list<HostArgs::Need> needs) {
    CtxLock lk;
    if (require_ready() || h.check(needs)) return 1;
    if (log_n > 30 || in_log_n > log_n) return fail("ntt: bad sizes");
    return by_field(field, [&](auto p) { return ntt_host<decltype(p)>(field, mode, a_in, in_log_n, log_n, omega, zeta, divisor, out_len, out, h); });
}
extern "C" int h2_ntt(int field, void *a, const void *omega, uint32_t log_n, int repr) {
    return ntt_host_dispatch(field, 0, a, log_n, log_n, omega, nullptr, nullptr, (size_t)1 << log_n, a, {"h2_ntt", repr}, {{a, "a"}, {omega, "omega"}});
}
extern "C" int h2_intt_scaled(int field, void *a, const void *omega_inv, const void *divisor, uint32_t log_n, int repr) {
    return ntt_host_dispatch(field, 1, a, log_n, log_n, omega_inv, nullptr, divisor, (size_t)1 << log_n, a, {"h2_intt_scaled", repr},
                             {{a, "a"}, {omega_inv, "omega_inv"}, {divisor, "divisor"}});
}
extern "C" int h2_coeff_to_extended(int field, const void *a, uint32_t k, uint32_t ext_k, const void *zeta, const void *ext_omega,
                                    void *out, int repr) {
    return ntt_host_dispatch(field, 2, a, k, ext_k, ext_omega, zeta, nullptr, (size_t)1 << ext_k, out, {"h2_coeff_to_extended", repr},
                             {{a, "a"}, {zeta, "zeta"}, {ext_omega, "ext_omega"}, {out, "out"}});
}
extern "C" int h2_extended_to_coeff(int field, const void *a, uint32_t ext_k, const void *ext_omega_inv, const void *ext_divisor,
                                    const void *zeta, size_t out_len, void *out, int repr) {
    return ntt_host_dispatch(field, 3, a, ext_k, ext_k, ext_omega_inv, zeta, ext_divisor, out_len, out, {"h2_extended_to_coeff", repr},
                             {{a, "a"}, {ext_omega_inv, "ext_omega_inv"}, {ext_divisor, "ext_divisor"}, {zeta, "zeta"}, {out, "out", out_len != 0}});
}
extern "C" int h2_ntt_dev(int field, const void *d_in, void *d_out, const void *omega, int omega_repr, uint32_t log_n, void *stream) {
    CtxLock lk;
    const HostArgs h("h2_ntt_dev", omega_repr);
    if (require_ready() || h.check({{omega, "omega"}})) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    StreamSplice splice(s);   // the twiddle cache, pow2 and the NTT scratch are the context's
    if (splice.failed) return 1;
    NttScales sc;   // Montgomery in, Montgomery out, no scaling
    return by_field(field, [&](auto p) {
        using P = decltype(p);
        return ntt_run<P>(field, (const fe *)d_in, log_n, (fe *)d_out, log_n, h.elem<P>(omega), sc, 1ull << log_n, s);
    });
}
// test / bench hook: 1 = the bulk-copy (TMA) persistent pass kernel where it applies, 0 = the classic kernel (default; ctx.cuh)
extern "C" int h2_test_set_ntt_tma(int on) {
    CtxLock lk;
    g_ctx.ntt_tma = on ? 1u : 0u;
    return 0;
}
extern "C" int h2_ntt_clear_cache(void) {
    CtxLock lk;
    if (require_ready()) return 1;
    cudaDeviceSynchronize();
    for (auto *t : g_ctx.twiddles) { t->buf.release(); delete t; }
    g_ctx.twiddles.clear();
    return 0;
}

int get_twiddles_any(int field, const fe &omega_mont, uint32_t log_n, cudaStream_t s, const fe **out) {
    return by_field(field, [&](auto p) { return get_twiddles<decltype(p)>(field, omega_mont, log_n, s, out); });
}

// ------------------------------------------------------------------------------------------------
// Device-resident polynomials (SURVEY.md section 8(f), row 3): the transforms and commits of the quotient
// pipeline without a PCIe round trip per call.  Data is kept in Montgomery form; every buffer has one spare
// slot so that a commit can append the blind.
// ------------------------------------------------------------------------------------------------
extern "C" int h2_poly_alloc(int field, size_t len, uint64_t *poly) {
    CtxLock lk;
    if (require_ready()) return 1;
    if (by_field(field, [](auto) { return 0; })) return 1;
    // A prover allocates and frees the same few sizes proof after proof: freed polynomials keep their device buffer in a small
    // pool, so that this is a memset on the stream instead of a cudaMalloc (and h2_poly_free no cudaFree + device sync).
    Context &X = g_ctx;
    PolyBuf *b = nullptr;
    for (size_t i = 0; i < X.poly_pool.size(); i++) {
        PolyBuf *c = X.poly_pool[i];
        if (c->buf.cap >= (len + 1) * sizeof(fe) && c->buf.cap <= (len + 1) * sizeof(fe) * 9 / 8 + 512) {
            b = c;
            X.poly_pool_bytes -= c->buf.cap;
            X.poly_pool.erase(X.poly_pool.begin() + i);
            break;
        }
    }
    if (!b) b = new PolyBuf();
    b->field = field; b->len = len;
    if (b->buf.ensure((len + 1) * sizeof(fe))) { delete b; return 1; }
    // zero-filled: a commit after a partial upload, or of a quotient shorter than the buffer, must not read stale memory
    if (cudaMemsetAsync(b->buf.p, 0, (len + 1) * sizeof(fe), X.stream) != cudaSuccess) { b->buf.release(); delete b; return fail("h2_poly_alloc: memset failed"); }
    uint64_t h = new_handle();
    X.polys[h] = b;
    *poly = h;
    return 0;
}
// Moves polynomials of the calling context into the shared registry, all or none (ctx.cuh: g_shared_polys).
extern "C" int h2_poly_share(const uint64_t *polys, size_t n) {
    CtxLock lk;
    if (require_ready()) return 1;
    if (n == 0) return 0;
    if (!polys) return fail("h2_poly_share: null handle array");
    Context &X = g_ctx;
    CU(cudaStreamSynchronize(X.stream));      // every write to them has landed before another context can read them
    std::lock_guard<std::mutex> reg(g_reg_mu);  // checked and moved under one lock: a shared handle cannot be freed in between
    for (size_t i = 0; i < n; i++)
        if (!X.polys.count(polys[i]) && !g_shared_polys.count(polys[i]))
            return fail("h2_poly_share: unknown polynomial handle (neither the calling context's nor shared)");
    for (size_t i = 0; i < n; i++) {
        auto it = X.polys.find(polys[i]);
        if (it == X.polys.end()) continue;    // already shared, or listed twice
        g_shared_polys[it->first] = it->second;
        X.polys.erase(it);
    }
    return 0;
}
// h2_poly_free of a polynomial the context X owned, taken out of X.polys (X's mutex held)
static int own_poly_free(Context &X, PolyBuf *b) {
    // every use of a resident polynomial is ordered on the context's stream, and so is its next owner's first write.
    // The pool is first-in first-out: when it is full the OLDEST buffers go (sizes an earlier workload left behind must not
    // pin the pool and push every later free onto the cudaFree + device-sync path, which would make a
    // replay after other work slower than the same replay in a fresh process)
    if (b->buf.cap > ((size_t)4 << 30)) {
        cudaSetDevice(X.device);
        cudaStreamSynchronize(X.stream);
        b->buf.release();
        delete b;
        return 0;
    }
    bool synced = false;
    while (!X.poly_pool.empty() && (X.poly_pool.size() >= 192 || X.poly_pool_bytes + b->buf.cap > ((size_t)4 << 30))) {
        PolyBuf *old = X.poly_pool.front();
        X.poly_pool.erase(X.poly_pool.begin());
        X.poly_pool_bytes -= old->buf.cap;
        if (!synced) { cudaSetDevice(X.device); cudaStreamSynchronize(X.stream); synced = true; }
        old->buf.release();
        delete old;
    }
    X.poly_pool.push_back(b);
    X.poly_pool_bytes += b->buf.cap;
    return 0;
}
extern "C" int h2_poly_free(uint64_t poly) {
    {
        CtxLock lk;
        Context &X = g_ctx;
        auto it = X.polys.find(poly);
        if (it != X.polys.end()) {
            PolyBuf *b = it->second;
            X.polys.erase(it);
            return own_poly_free(X, b);
        }
    }
    return shared_poly_free(poly);             // without this context's mutex: it may wait for calls on other lanes
}
int convert_field(int field, fe *d, size_t n, int to_mont, cudaStream_t s) {
    if (n == 0) return 0;
    return by_field(field, [&](auto p) {
        LAUNCH(convert_kernel<decltype(p)>, blocks_for(n, 256), 256, 0, s, d, (uint64_t)n, to_mont);
        return 0;
    });
}
extern "C" int h2_poly_upload(uint64_t poly, const void *src, size_t len, int repr) {
    CtxLock lk;
    const HostArgs h("h2_poly_upload", repr);
    if (require_ready() || h.check({{src, "src", len != 0}})) return 1;
    PolyArgs g("h2_poly_upload");
    PolyBuf *b = g.out(poly, "poly", len, "len");
    if (!b) return 1;
    cudaStream_t s = g_ctx.stream;
    if (h.up(b->field, b->buf.as<fe>(), src, len, s)) return 1;
    CU(cudaStreamSynchronize(s));      // src may be pageable
    return 0;
}
// a[index] += delta: the one-coefficient corrections of the opening argument (poly/commitment/prover.rs:51 `s_poly[0] -= s_at_x3`,
// :78 `p_prime_poly[0] -= v`) on a resident polynomial
template <class P> __global__ void poly_add_at_kernel(fe *a, fe delta_mont) { fe_store(a, fe_add<P>(fe_load(a), delta_mont)); }
extern "C" int h2_poly_add_at(uint64_t poly, size_t index, const void *delta, int repr) {
    CtxLock lk;
    const HostArgs h("h2_poly_add_at", repr);
    if (require_ready() || h.check({{delta, "delta"}})) return 1;
    PolyArgs g("h2_poly_add_at");
    PolyBuf *b = g.out(poly, "poly", 0, "0");
    if (!b) return 1;
    if (index >= b->len) return fail("h2_poly_add_at: index out of range");
    cudaStream_t s = g_ctx.stream;
    return by_field(b->field, [&](auto p) {
        using P = decltype(p);
        LAUNCH(poly_add_at_kernel<P>, 1, 1, 0, s, b->buf.as<fe>() + index, h.elem<P>(delta));
        return 0;
    });
}
// dst[dst_off .. dst_off + len) = src[src_off .. src_off + len) on the device: the h(X) pieces (plonk/vanishing/prover.rs:95-100
// `h_poly.chunks_exact(n)`), or a copy of a column that an in-place step is about to overwrite
extern "C" int h2_poly_copy(uint64_t dst, size_t dst_off, uint64_t src, size_t src_off, size_t len) {
    CtxLock lk;
    if (require_ready()) return 1;
    PolyArgs g("h2_poly_copy");
    PolyBuf *d = g.out(dst, "dst", dst_off, len, "dst_off + len");
    if (!d) return 1;
    PolyBuf *a = g.in(src, "src", src_off, len, "src_off + len");
    if (!a) return 1;
    if (d == a && !(dst_off + len <= src_off || src_off + len <= dst_off)) return fail("h2_poly_copy: overlapping ranges");
    if (len) CU(cudaMemcpyAsync(d->buf.as<fe>() + dst_off, a->buf.as<fe>() + src_off, len * sizeof(fe), cudaMemcpyDeviceToDevice, g_ctx.stream));
    return 0;
}
extern "C" int h2_poly_download(uint64_t poly, void *dst, size_t len, int repr) {
    CtxLock lk;
    const HostArgs h("h2_poly_download", repr);
    if (require_ready() || h.check({{dst, "dst", len != 0}})) return 1;
    PolyArgs g("h2_poly_download");
    PolyBuf *b = g.in(poly, "poly", len, "len");
    if (!b) return 1;
    return h.down(b->field, dst, b->buf.as<fe>(), len, g_ctx.stream);
}
// h2_poly_upload_dev / h2_poly_download_dev (K25, columns_io.cuh): column i moves lens[i] elements between polys[i] and the
// caller's device pointer ptrs[i], every column in one launch on the caller's stream.  Every check runs before the first
// launch; the caller's pointers are checked where they are non-empty.
static int poly_io_dev(const char *who, bool up, const uint64_t *polys, size_t count, const void *const *ptrs, const size_t *lens, int repr,
                       void *stream) {
    const char *pname = up ? "d_src" : "d_dst";
    CtxLock lk;
    const HostArgs h(who, repr);
    if (require_ready() || h.check({{polys, "polys", count != 0}, {ptrs, pname, count != 0}, {lens, "lens", count != 0}})) return 1;
    if (count == 0) return 0;
    Context &X = g_ctx;
    const std::string w(who);
    auto bad = [&](size_t i, const std::string &why) { return fail(w + ": " + pname + "[" + std::to_string(i) + "]: " + why); };
    PolyArgs g(who);
    std::vector<PolyBuf *> ps;
    if ((up ? g.out(polys, count, "polys", lens, "lens", ps) || g.distinct() : g.in(polys, count, "polys", lens, "lens", ps))) return 1;
    uint64_t longest = 0;
    std::vector<IoCol> io(count);
    std::vector<std::pair<uintptr_t, size_t>> ranges;   // download: the caller's byte ranges, to refuse overlaps
    for (size_t i = 0; i < count; i++) {
        io[i] = {(uint64_t)(uintptr_t)ptrs[i], (uint64_t)lens[i]};
        if (lens[i] == 0) continue;
        if (!ptrs[i]) return bad(i, "null pointer");
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, ptrs[i]) != cudaSuccess) { cudaGetLastError(); a.type = cudaMemoryTypeUnregistered; }
        if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged)
            return bad(i, std::string("not device memory (host columns go through ") + (up ? "h2_poly_upload)" : "h2_poly_download)"));
        if (a.device != X.device)
            return bad(i, "memory of device " + std::to_string(a.device) + ", not the calling context's device " + std::to_string(X.device));
        if ((uintptr_t)ptrs[i] % 16) return bad(i, "not 16-byte aligned");
        if (!up) ranges.push_back({(uintptr_t)ptrs[i], i});
        if (lens[i] > longest) longest = lens[i];
    }
    if (!up) {
        std::sort(ranges.begin(), ranges.end());
        size_t reach = 0;   // of the ranges so far (by start address), the one that ends last
        for (size_t j = 1; j < ranges.size(); j++) {
            const size_t prev = ranges[reach].second, cur = ranges[j].second;
            if (ranges[j].first < ranges[reach].first + lens[prev] * sizeof(fe))
                return bad(std::max(prev, cur), "overlaps " + std::string(pname) + "[" + std::to_string(std::min(prev, cur)) + "]");
            reach = j;   // no overlap: range j starts at or after every earlier end, so it ends last
        }
    }
    if (longest == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    StreamSplice splice(s);   // the column table is the context's scratch
    if (splice.failed) return 1;
    ColTable t;
    if (col_table(ps, io.data(), count * sizeof(IoCol), s, &t)) return 1;
    return by_field(ps[0]->field, [&](auto p) {
        using P = decltype(p);
        for (size_t c0 = 0; c0 < count; c0 += 65535) {   // grid.y limit
            const uint32_t cols = (uint32_t)std::min<size_t>(count - c0, 65535);
            LAUNCH(columns_io_kernel<P>, dim3(blocks_for(longest, 256), cols), 256, 0, s, t.cols, reinterpret_cast<const IoCol *>(t.data), (uint32_t)c0,
                   up ? 1 : 0, h.canon() ? 1 : 0);
        }
        return 0;
    });
}
extern "C" int h2_poly_upload_dev(const uint64_t *polys, size_t count, const void *const *d_src, const size_t *lens, int repr, void *stream) {
    return poly_io_dev("h2_poly_upload_dev", true, polys, count, d_src, lens, repr, stream);
}
extern "C" int h2_poly_download_dev(const uint64_t *polys, size_t count, void *const *d_dst, const size_t *lens, int repr, void *stream) {
    return poly_io_dev("h2_poly_download_dev", false, polys, count, (const void *const *)d_dst, lens, repr, stream);
}
// mode as in ntt_host: 1 = inverse transform with divisor, 2 = coeff_to_extended, 3 = extended_to_coeff.  Column i goes from
// src[i] to dst[i]; a batch reaches ntt_run through one table of its columns' pointers (the sources, then the destinations).
template <class P>
static int poly_transform(const std::vector<PolyBuf *> &dst, const std::vector<PolyBuf *> &src, int mode, uint32_t in_log_n, uint32_t log_n,
                          const void *omega, const void *zeta, const void *divisor, size_t out_len, const HostArgs &h) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const size_t count = dst.size();
    const NttScales sc = host_scales<P>(h, false, mode, zeta, divisor);   // resident data: Montgomery in and out
    if (count == 1) {
        if (ntt_run<P>(P::ID, src[0]->buf.as<fe>(), in_log_n, dst[0]->buf.as<fe>(), log_n, h.elem<P>(omega), sc, out_len, s)) return 1;
    } else {
        std::vector<PolyBuf *> cols(src);
        cols.insert(cols.end(), dst.begin(), dst.end());
        ColTable t;
        if (col_table(cols, nullptr, 0, s, &t) ||
            ntt_run<P>(P::ID, nullptr, in_log_n, nullptr, log_n, h.elem<P>(omega), sc, out_len, s, count, t.cols, t.cols + count))
            return 1;
    }
    return 0;   // asynchronous: later calls are ordered behind it on the stream
}
static int poly_transform_dispatch(uint64_t dst, uint64_t src, int mode, uint32_t in_log_n, uint32_t log_n, const void *omega, const void *zeta,
                                   const void *divisor, size_t out_len, const HostArgs &h, std::initializer_list<HostArgs::Need> needs,
                                   const char *in_name, const char *out_name) {
    const char *who = h.who;
    CtxLock lk;
    if (require_ready() || h.check(needs)) return 1;
    if (log_n > 30 || in_log_n > log_n) return fail("ntt: bad sizes");
    if (out_len > ((size_t)1 << log_n)) out_len = (size_t)1 << log_n;
    PolyArgs g(who);
    PolyBuf *d = g.out(dst, "dst", out_len, out_name);
    if (!d) return 1;
    PolyBuf *a = g.in(src, "src", (size_t)1 << in_log_n, in_name);
    if (!a) return 1;
    if (d == a && out_len != ((size_t)1 << log_n)) return fail(std::string(who) + ": in place needs out_len == 2^log_n");
    if (d == a && in_log_n != log_n) return fail(std::string(who) + ": in place needs equal input and output sizes");
    return by_field(a->field, [&](auto p) { return poly_transform<decltype(p)>({d}, {a}, mode, in_log_n, log_n, omega, zeta, divisor, out_len, h); });
}
// `count` columns of one size and domain, dst[i] = transform(src[i]); every check runs before the first launch.  A destination
// listed twice, or that is another column's source, would race with that column's launch; dst[i] == src[i] works in place
// where the sizes are equal, as in the one-column call.  Errors name the first offending index.
static int poly_transform_batch(const uint64_t *dst, const uint64_t *src, size_t count, int mode, uint32_t in_log_n, uint32_t log_n,
                                const void *omega, const void *zeta, const void *divisor, const HostArgs &h,
                                std::initializer_list<HostArgs::Need> needs, const char *in_name, const char *out_name) {
    const std::string who = h.who;
    CtxLock lk;
    if (require_ready() || h.check(needs)) return 1;
    if (log_n > 30 || in_log_n > log_n) return fail(who + ": bad sizes");
    if (count == 0) return 0;
    if (!dst || !src) return fail(who + ": null handle array");
    const size_t n_in = (size_t)1 << in_log_n, n_out = (size_t)1 << log_n;
    PolyArgs g(h.who);
    std::vector<PolyBuf *> d, a;
    if (g.out(dst, count, "dst", n_out, out_name, d) || g.in(src, count, "src", n_in, in_name, a) || g.distinct("dst", "src")) return 1;
    for (size_t i = 0; i < count; i++)
        if (d[i] == a[i] && in_log_n != log_n)
            return fail(who + ": dst[" + std::to_string(i) + "] == src[" + std::to_string(i) + "]: in place needs equal input and output sizes");
    return by_field(d[0]->field, [&](auto p) { return poly_transform<decltype(p)>(d, a, mode, in_log_n, log_n, omega, zeta, divisor, n_out, h); });
}
extern "C" int h2_poly_lagrange_to_coeff(uint64_t dst, uint64_t src, uint32_t k, const void *omega_inv, const void *divisor, int repr) {
    return poly_transform_dispatch(dst, src, 1, k, k, omega_inv, nullptr, divisor, (size_t)1 << k, {"h2_poly_lagrange_to_coeff", repr},
                                   {{omega_inv, "omega_inv"}, {divisor, "divisor"}}, "2^k", "2^k");
}
extern "C" int h2_poly_coeff_to_extended(uint64_t dst, uint64_t src, uint32_t k, uint32_t ext_k, const void *zeta, const void *ext_omega, int repr) {
    return poly_transform_dispatch(dst, src, 2, k, ext_k, ext_omega, zeta, nullptr, (size_t)1 << ext_k, {"h2_poly_coeff_to_extended", repr},
                                   {{zeta, "zeta"}, {ext_omega, "ext_omega"}}, "2^k", "2^ext_k");
}
extern "C" int h2_poly_extended_to_coeff(uint64_t dst, uint64_t src, uint32_t ext_k, const void *ext_omega_inv, const void *ext_divisor,
                                         const void *zeta, size_t out_len, int repr) {
    return poly_transform_dispatch(dst, src, 3, ext_k, ext_k, ext_omega_inv, zeta, ext_divisor, out_len, {"h2_poly_extended_to_coeff", repr},
                                   {{ext_omega_inv, "ext_omega_inv"}, {ext_divisor, "ext_divisor"}, {zeta, "zeta"}}, "2^ext_k", "out_len");
}
extern "C" int h2_poly_lagrange_to_coeff_batch(const uint64_t *dst, const uint64_t *src, size_t count, uint32_t k, const void *omega_inv,
                                               const void *divisor, int repr) {
    return poly_transform_batch(dst, src, count, 1, k, k, omega_inv, nullptr, divisor, {"h2_poly_lagrange_to_coeff_batch", repr},
                                {{omega_inv, "omega_inv", count != 0}, {divisor, "divisor", count != 0}}, "2^k", "2^k");
}
extern "C" int h2_poly_coeff_to_extended_batch(const uint64_t *dst, const uint64_t *src, size_t count, uint32_t k, uint32_t ext_k, const void *zeta,
                                               const void *ext_omega, int repr) {
    return poly_transform_batch(dst, src, count, 2, k, ext_k, ext_omega, zeta, nullptr, {"h2_poly_coeff_to_extended_batch", repr},
                                {{zeta, "zeta", count != 0}, {ext_omega, "ext_omega", count != 0}}, "2^k", "2^ext_k");
}
// rows [start, start + rows) of column c <- vals[c rows ..], from `repr` into Montgomery form on the way
template <class P> __global__ void set_rows_kernel(fe *const *cols, const fe *vals, uint64_t start, uint64_t rows, uint64_t total, int canon) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    fe x = fe_load(vals + i);
    if (canon) x = fe_to_mont<P>(x);
    fe_store(cols[i / rows] + start + i % rows, x);
}
extern "C" int h2_poly_set_rows(const uint64_t *polys, size_t count, size_t start, size_t rows, const void *values, int repr) {
    static const char *who = "h2_poly_set_rows";
    CtxLock lk;
    const HostArgs h(who, repr);
    if (require_ready() || h.check({{values, "values", count != 0 && rows != 0}})) return 1;
    if (count == 0) return 0;
    if (!polys) return fail(std::string(who) + ": null handle array");
    // the column table, count pointers in (count + 3) / 4 elements and then count x rows values, must fit in size_t
    if (rows != 0 && count > ((size_t)-1 / sizeof(fe) - (count + 3) / 4) / rows) return fail(std::string(who) + ": count * rows overflows");
    PolyArgs g(who);
    std::vector<PolyBuf *> ps;
    if (g.out(polys, count, "polys", start, rows, "start + rows", ps) || g.distinct()) return 1;
    if (rows == 0) return 0;
    const size_t total = count * rows;
    cudaStream_t s = g_ctx.stream;
    ColTable t;
    if (col_table(ps, values, total * sizeof(fe), s, &t)) return 1;
    return by_field(ps[0]->field, [&](auto p) {
        LAUNCH(set_rows_kernel<decltype(p)>, blocks_for(total, 256), 256, 0, s, t.cols, (const fe *)t.data, (uint64_t)start, (uint64_t)rows,
               (uint64_t)total, h.canon() ? 1 : 0);
        return 0;
    });
}
// The vanishing argument's quotient (plonk/vanishing/prover.rs:84-100, K24): pieces[i] = coefficients [i n, (i + 1) n) of
// extended_to_coeff(divide_by_vanishing_poly(src)), in one transform.  The division rides on the first pass's loads
// (NTT_IN_TABLE, t_evals after the column table in one upload), the ζ un-shift, 1 / 2^ext_k and the split on the last
// pass's stores (NTT_OUT_PIECES); src is only read.
extern "C" int h2_poly_vanishing_quotient(const uint64_t *pieces, size_t count, uint64_t src, uint32_t k, uint32_t ext_k,
                                          const void *ext_omega_inv, const void *ext_divisor, const void *zeta, const void *t_evals,
                                          uint32_t t_len, int repr) {
    static const char *who = "h2_poly_vanishing_quotient";
    CtxLock lk;
    const HostArgs h(who, repr);
    if (require_ready() || h.check({{ext_omega_inv, "ext_omega_inv"}, {ext_divisor, "ext_divisor"}, {zeta, "zeta"}, {t_evals, "t_evals"}}))
        return 1;
    if (const char *why = vanishing_quotient_sizes(k, ext_k, count, t_len)) return fail(std::string(who) + ": " + why);
    if (!pieces) return fail(std::string(who) + ": null handle array");
    PolyArgs g(who);
    std::vector<PolyBuf *> d;
    PolyBuf *a = nullptr;
    if (g.out(pieces, count, "pieces", (size_t)1 << k, "2^k", d) || !(a = g.in(src, "src", (size_t)1 << ext_k, "2^ext_k")) || g.distinct())
        return 1;
    cudaStream_t s = g_ctx.stream;
    ColTable t;
    if (col_table(d, t_evals, (size_t)t_len * sizeof(fe), s, &t) || h.to_mont(a->field, t.data, t_len, s)) return 1;
    return by_field(a->field, [&](auto p) {
        using P = decltype(p);
        NttScales sc = host_scales<P>(h, false, 3, zeta, ext_divisor);   // extended_to_coeff's: Montgomery in and out
        sc.in_table = t.data; sc.in_mask = t_len - 1;
        sc.pieces = true; sc.piece_log = k;
        return ntt_run<P>(P::ID, a->buf.as<fe>(), ext_k, nullptr, ext_k, h.elem<P>(ext_omega_inv), sc, (uint64_t)count << k, s, 1, nullptr, t.cols);
    });
}
