// C ABI of the engine, part 2 of 5: the MSM pipeline (msm.cuh, fixedbase.cuh), resident base sets, the IPA round loop (ipa.cuh).
// up to this many references the accumulation runs a pair / quad of lanes per work item; fixed-base passes (few, short buckets: the kernel lasts
// as long as its longest chain) up to twice that
#define H2_MSM_QUAD_ACCUM_REFS (g_ctx.small_accum_refs)
#include "util_kernels.cuh"
#include "msm.cuh"
#include "ipa.cuh"
#include "ntt.cuh"
#include "ecfft.cuh"
#include "fixedbase.cuh"

// What an MSM pass runs on: a registered set's digit-multiples table (mode 2, H2_FB_BITS) or window table (mode 1, window c, `stride`
// points per window), or plain bases (mode 0, window c; 0: chosen by size)
struct PassBases { const affine *bases; uint32_t c = 0, mode = 0; uint64_t stride = 0; };
static PassBases pass_bases(const BaseSet *b) {
    if (b->dtable.p) return {b->dtable.as<affine>(), H2_FB_BITS, 2, b->n};
    if (b->table.p) return {b->table.as<affine>(), b->c, 1, b->n};
    return {b->buf.as<affine>()};
}


// ------------------------------------------------------------------------------------------------
// MSM pipeline
// ------------------------------------------------------------------------------------------------
static int exclusive_scan_u32(uint32_t *d, uint64_t n, cudaStream_t s, const uint32_t *only_if = nullptr) {
    const uint64_t per_block = (uint64_t)H2_SCAN_BLOCK * H2_SCAN_ITEMS;
    uint32_t nb = (uint32_t)((n + per_block - 1) / per_block);
    if (g_ctx.scan_blocks.ensure((size_t)nb * 4 + 16)) return 1;
    uint32_t *bs = g_ctx.scan_blocks.as<uint32_t>();
    LAUNCH(scan_block_sums_kernel, nb, H2_SCAN_BLOCK, 0, s, d, n, bs, only_if);
    LAUNCH(scan_single_block_kernel, 1, H2_SCAN_BLOCK, 0, s, bs, nb, only_if);
    LAUNCH(scan_apply_kernel, nb, H2_SCAN_BLOCK, 0, s, d, n, bs, only_if);
    return 0;
}

// Arrival of the inputs of a one-shot MSM in `k` chunks (events on the copy stream): chunk j = points
// [chunk_first(n, k, j), chunk_first(n, k, j + 1)).  The chunks GROW: nothing can run before the first chunk has
// landed, so it is small (1/16 - 1/4 of the points), and the accumulation of chunk j hides the upload of the larger
// chunk j + 1 -- the link stays busy from t = 0 and the GPU from the first chunk's arrival.  (Equal chunks leave the
// GPU idle for 1/k of the upload time.)
uint32_t g_chunk_cut[H2_MAX_UPLOAD_CHUNKS + 1][H2_MAX_UPLOAD_CHUNKS + 1] = {
    {0, 16, 16, 16, 16}, {0, 16, 16, 16, 16}, {0, 4, 16, 16, 16}, {0, 2, 8, 16, 16}, {0, 1, 4, 10, 16}};   // sixteenths (h2_test_set_chunk_cuts)
static inline size_t chunk_first(size_t n, uint32_t k, uint32_t j) {
    const auto &cut = g_chunk_cut;
    if (k > H2_MAX_UPLOAD_CHUNKS) k = H2_MAX_UPLOAD_CHUNKS;
    if (j >= k) return n;
    return (size_t)((unsigned __int128)n * cut[k][j] / 16);
}

// A fixed-base MSM over resident bases is launched with the same parameters call after call: the second call with a given
// key is captured into a CUDA graph, later ones replay it.
static int msm_issue_or_replay(const std::function<int()> &issue, bool graphable, const void *d_scalars, const void *d_bases, const void *d_out,
                               size_t n, uint64_t stride, uint32_t c, uint32_t sets, int scalars_mont, int out_canonical, bool fast, cudaStream_t s) {
    Context &X = g_ctx;
    if (!(graphable && X.graphs_on && !g_prof_on)) return issue();
    MsmGraph *ge = nullptr;
    for (auto &e : X.graphs)
        if (e.scalars == d_scalars && e.bases == d_bases && e.out == d_out && e.n == n && e.stride == stride && e.c == c && e.sets == sets &&
            e.scalars_mont == scalars_mont && e.out_canonical == out_canonical && e.fast == (fast ? 1u : 0u)) { ge = &e; break; }
    if (ge && ge->gen != g_alloc_gen) {   // some buffer moved since the capture
        if (ge->exec) cudaGraphExecDestroy(ge->exec);
        ge->exec = nullptr; ge->seen = 0; ge->gen = g_alloc_gen;
    }
    if (!ge) {
        if (X.graphs.size() >= 16) {   // evict the least recently used entry
            size_t v = 0;
            for (size_t i = 1; i < X.graphs.size(); i++) if (X.graphs[i].stamp < X.graphs[v].stamp) v = i;
            if (X.graphs[v].exec) cudaGraphExecDestroy(X.graphs[v].exec);
            X.graphs.erase(X.graphs.begin() + v);
        }
        MsmGraph e;
        e.scalars = d_scalars; e.bases = d_bases; e.out = d_out; e.n = n; e.stride = stride; e.gen = g_alloc_gen; e.c = c; e.sets = sets;
        e.scalars_mont = scalars_mont; e.out_canonical = out_canonical; e.fast = fast ? 1u : 0u;
        X.graphs.push_back(e);
        ge = &X.graphs.back();
    }
    ge->stamp = ++X.graph_stamp;
    if (ge->exec) {
        CU(cudaGraphLaunch(ge->exec, s));
        g_launches.fetch_add(ge->launches, std::memory_order_relaxed);
        return 0;
    }
    if (ge->seen++ == 0) return issue();     // first sighting: run eagerly (the buffers may still be growing)
    const uint64_t l0 = g_launches.load();
    if (cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); return issue(); }
    int rc = issue();
    cudaGraph_t graph = nullptr;
    cudaError_t ce = cudaStreamEndCapture(s, &graph);
    if (rc || ce != cudaSuccess || !graph) {
        if (graph) cudaGraphDestroy(graph);
        cudaGetLastError();
        ge->seen = 0;
        // Nothing captured has run, so run eagerly.  The failure need not be this call's: a device-wide synchronisation on
        // another thread (another lane's cudaFree, cudaDeviceSynchronize, ...) invalidates a capture in progress, and then
        // every later call of the capture fails.  An error of the pass itself comes back from the eager run.
        return issue();
    }
    ge->launches = g_launches.load() - l0;
    ce = cudaGraphInstantiate(&ge->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ce != cudaSuccess) { ge->exec = nullptr; cudaGetLastError(); return issue(); }
    CU(cudaGraphLaunch(ge->exec, s));
    return 0;
}

// fixed != 0: d_bases is a window table (stride points per window) built with window size c.
// bc != nullptr: the bases arrive chunk by chunk while this runs.  Each chunk is then sorted and accumulated on its own
// (own bins, work items and bucket sums) as soon as it has landed, and the bucket reduce adds the per-chunk bucket sums:
// the upload of all but the first chunk hides behind the accumulation.
// fast: a pass over a window table with bins and without chunks may run without its fallback kernels (MsmPlan::fast); *ran_fast (if
// given) tells whether it did, and then its result is valid only if both device flags come back clear (msm_pass).  rerun: the pass
// re-runs, in full, a fast one whose flags came back set.
template <class P, class PS>
static int msm_run(const fe *d_scalars, int scalars_mont, const affine *d_bases, size_t n, uint32_t c, uint32_t fixed, uint64_t stride,
                   jacobian *d_out, int out_canonical, cudaStream_t s, const BasesChunks *bc, uint32_t sets, bool fast, bool rerun,
                   bool *ran_fast) {
    Context &X = g_ctx;
    if (ran_fast) *ran_fast = false;
    if (n == 0) {   // empty sum = identity, one per scalar vector
        jacobian id;
        id.x = fe_zero(); id.y = out_canonical ? fe_zero() : fe_one<P>(); id.z = fe_zero();
        if (out_canonical) id.y.v[0] = 1;
        std::vector<jacobian> ids(sets ? sets : 1u, id);
        CU(cudaMemcpyAsync(d_out, ids.data(), ids.size() * sizeof id, cudaMemcpyHostToDevice, s));
        CU(cudaStreamSynchronize(s));
        return 0;
    }
    std::function<int()> issue;
    // h2_test_last_msm_plan: mode, c, W, sets, accumulation, natural, fast, re-run of a fast pass -- recorded here on the host,
    // so a pass replayed from a captured graph reports the same
    auto record = [&X, rerun](uint32_t mode, uint32_t c_, uint32_t W, uint32_t sets_, uint32_t accum, uint32_t natural, uint32_t fast_) {
        const uint32_t v[8] = {mode, c_, W, sets_, accum, natural, fast_, rerun ? 1u : 0u};
        memcpy(X.last_plan, v, sizeof v);
        X.have_plan = true;
    };
    if (fixed == 2) {   // direct sum over the digit-multiples table (fixedbase.cuh): accumulate + reduce tree
        FbPlan fp;
        fp.total = n; fp.sets = sets ? sets : 1u; fp.split = fb_split(n, fp.sets); fp.scalars_mont = scalars_mont ? 1u : 0u;
        record(2, H2_FB_BITS, H2_FB_WINDOWS, fp.sets, 2, 0, 0);
        const uint64_t count0 = n * fp.split;
        if (X.fb_a.ensure(fp.sets * count0 * sizeof(xyzz)) || X.fb_b.ensure(fp.sets * fb_ctas(count0, fb_fan(count0)) * sizeof(xyzz))) return 1;
        issue = [&X, fp, count0, d_scalars, d_bases, d_out, out_canonical, s]() -> int {
            auto k_acc = fb_accum_kernel<P, PS>;
            auto k_red = fb_reduce_kernel<P, PS>;
            xyzz *a = X.fb_a.as<xyzz>(), *b = X.fb_b.as<xyzz>();
            prof_begin(PROF_MSM_ACCUM0, s);
            LAUNCH(k_acc, blocks_for(fp.sets * count0, 128), 128, 0, s, fp, d_scalars, d_bases, a);
            prof_end(s);
            uint64_t count = count0, in_stride = count0;
            for (;;) {
                const uint32_t f = fb_fan(count);
                const uint64_t ctas = fb_ctas(count, f);
                LAUNCH(k_red, dim3((unsigned)ctas, fp.sets), 4 * H2_FB_QUADS, 0, s, (const xyzz *)a, count, in_stride, f, b, ctas,
                       ctas == 1 ? d_out : (jacobian *)nullptr, (uint32_t)out_canonical);
                if (ctas == 1) break;
                xyzz *t = a; a = b; b = t;
                count = ctas; in_stride = ctas;
            }
            return 0;
        };
        return msm_issue_or_replay(issue, !bc, d_scalars, d_bases, d_out, n, stride, H2_FB_BITS, fp.sets, scalars_mont, out_canonical, fast, s);
    }
    const uint32_t glv = (!fixed && X.glv_on && n < (1ull << 30)) ? 1u : 0u;
    if (c == 0) c = X.window_override ? X.window_override : msm_default_window(n, glv);
    if (c > 24) return fail("msm: window bits > 24");
    const uint32_t K = (bc && !fixed && bc->k > 1) ? bc->k : 1u;
    const uint32_t force_cap = X.sort_bins ? 0u : H2_MSM_NO_BINS;
    MsmPlan p;                       // the whole problem: bucket reduce and window combine
    msm_make_plan(p, n, c, 0, 0, fixed, stride, glv, sets, force_cap);
    p.chunks = K;
    p.fast = (fixed == 1 && !bc && fast && p.cap != 0) ? 1u : 0u;
    if (ran_fast) *ran_fast = p.fast != 0;
    // ... whose work items are whole buckets: with T >= the bin capacity a bucket can only exceed T by overflowing its bin, so
    // "a bucket was split" (flags[0], ~5 buckets of a k = 14 commit at T = 32) never fails a pass that the sort flag would not
    if (p.fast && p.T < p.cap) { p.T = p.cap; p.acc_chunk[0] = p.T; }
    p.natural = (p.fast && p.G <= X.natural_max_buckets && p.max_refs <= 2 * H2_MSM_QUAD_ACCUM_REFS && (X.accum_ways <= 1 || X.accum_ways >= 12)) ? 1u : 0u;
    MsmPlan pk[H2_MAX_UPLOAD_CHUNKS];   // one chunk of points: sort, work items, accumulation
    size_t first[H2_MAX_UPLOAD_CHUNKS + 1];
    for (uint32_t j = 0; j <= K; j++) first[j] = chunk_first(n, K, j);
    uint64_t ref_space = 0, max_items = 0, part_total = 0;
    uint32_t t_max = 0;
    for (uint32_t j = 0; j < K; j++) {
        if (K == 1) pk[0] = p;
        else msm_make_plan(pk[j], first[j + 1] - first[j], c, 0, 0, fixed, stride, glv, sets, force_cap);
        if (pk[j].ref_space >= (1ull << 32)) return fail("msm: n * windows exceeds 2^32 references");
        ref_space = pk[j].ref_space > ref_space ? pk[j].ref_space : ref_space;
        max_items = pk[j].max_items > max_items ? pk[j].max_items : max_items;
        part_total = pk[j].part_total > part_total ? pk[j].part_total : part_total;
        t_max = pk[j].T > t_max ? pk[j].T : t_max;
    }
    bool thread_per_item = false;   // the accumulation's branch below, for any chunk
    for (uint32_t j = 0; j < K; j++) thread_per_item |= pk[j].max_refs > (pk[j].fixed ? 2 : 1) * H2_MSM_QUAD_ACCUM_REFS;
    record(fixed, c, p.W, p.sets, thread_per_item ? 1u : 0u, p.natural, p.fast);
    // batched-affine rounds ahead of the XYZZ chain (msm.cuh K4a) for the throughput-bound sizes: every chunk plans its own
    // chunk's rounds; their level arrays (56 B per reference over the rounds, per chunk) may take at most half of the free
    // device memory -- a larger problem runs without them
    uint64_t ba_space = 0;
    if (!fixed && X.ba_rounds) {
        size_t free_b = 0, total_b = 0;
        CU(cudaMemGetInfo(&free_b, &total_b));
        for (uint32_t j = 0; j < K; j++) {
            if (pk[j].max_refs > H2_MSM_QUAD_ACCUM_REFS && (uint64_t)K * pk[j].ref_space * 56 <= free_b / 2) msm_plan_ba(pk[j], X.ba_rounds, X.ba_target);
            if (pk[j].ba) ba_space = pk[j].ref_space > ba_space ? pk[j].ref_space : ba_space;
        }
    }
    if (K == 1) p.ba = pk[0].ba;
    if (ba_space)
        for (uint32_t r = 0; r < H2_BA_MAX_ROUNDS; r++)
            if (X.ba_lv[r].ensure(K * ((ba_space >> (r + 1)) + 1) * sizeof(affine))) return 1;
    if (glv && (X.bases_phi.ensure(n * sizeof(affine)) || X.glv_parts.ensure(n * 32))) return 1;
    if (fixed && (uint64_t)p.W * stride >= (1ull << 31)) return fail("msm: window table too large for 31-bit references");
    if (p.G >= (1ull << 32) || n >= (1ull << 31)) return fail("msm: n * windows exceeds 2^32 references");
    if (scalars_mont && X.scal_canon.ensure(n * p.sets * sizeof(fe))) return 1;
    const size_t small_words = 2 * (t_max + 2) + 8;   // size_hist (T + 2) | size_cursor (T + 1) | flags
    part_total += 1;
    if (X.counts.ensure(K * (p.G + 1) * 4) || X.cursor.ensure(K * 2 * p.G * 4) || X.refs.ensure(K * ref_space * 4) ||
        X.size_hist.ensure(K * small_words * 4) || X.items.ensure(K * max_items * sizeof(uint2)) ||
        X.bucket_sum.ensure(K * p.G * sizeof(xyzz)) || X.pkey.ensure(K * part_total * 4) || X.pstart.ensure(K * part_total * 4) ||
        X.pend.ensure(K * part_total * 4) || X.ppt.ensure(K * part_total * sizeof(xyzz)) ||
        X.ra_t.ensure((size_t)p.Wb * p.m1 * sizeof(xyzz)) || X.ra_e.ensure((size_t)p.Wb * p.m1 * sizeof(xyzz)) ||
        X.r0.ensure((size_t)p.Wb * p.nb0 * H2_R0_ROWS * sizeof(xyzz)) || X.r1.ensure((size_t)p.Wb * p.r1_rows * sizeof(xyzz)) ||
        X.wsum.ensure((size_t)p.Wb * sizeof(xyzz)))
        return 1;
    MsmBuffers Mk[H2_MAX_UPLOAD_CHUNKS];
    for (uint32_t j = 0; j < K; j++) {
        MsmBuffers &M = Mk[j];
        const size_t o = first[j];
        M.scalars = d_scalars + o; M.bases = d_bases + o; M.bases_phi = X.bases_phi.as<affine>() + o;
        M.glv_parts = X.glv_parts.as<uint32_t>() + 8 * o; M.scalars_mont = scalars_mont ? 1u : 0u;
        M.scal_canon = X.scal_canon.as<fe>() + o;
        M.counts = X.counts.as<uint32_t>() + j * (p.G + 1); M.cursor = X.cursor.as<uint32_t>() + j * 2 * p.G; M.cursor2 = M.cursor + p.G;
        M.refs = X.refs.as<uint32_t>() + j * ref_space;
        M.size_hist = X.size_hist.as<uint32_t>() + j * small_words; M.size_cursor = M.size_hist + (pk[j].T + 2); M.flags = M.size_cursor + (pk[j].T + 2);
        M.items = X.items.as<uint2>() + j * max_items;
        M.bucket_sum = X.bucket_sum.as<xyzz>() + j * p.G;
        for (uint32_t r = 0; r < H2_BA_MAX_ROUNDS; r++) M.ba[r] = ba_space ? X.ba_lv[r].as<affine>() + j * ((ba_space >> (r + 1)) + 1) : nullptr;
        M.pkey = X.pkey.as<uint32_t>() + j * part_total; M.pstart = X.pstart.as<uint32_t>() + j * part_total;
        M.pend = X.pend.as<uint32_t>() + j * part_total; M.ppt = X.ppt.as<xyzz>() + j * part_total;
        M.ra_t = X.ra_t.as<xyzz>(); M.ra_e = X.ra_e.as<xyzz>(); M.r0 = X.r0.as<xyzz>(); M.r1 = X.r1.as<xyzz>();
        M.wsum = X.wsum.as<xyzz>(); M.result = d_out;
    }
    X.last_flags = Mk[0].flags;

    {   // scratch of the scan (sized here so that nothing allocates while a graph is being captured)
        const uint64_t per_block = (uint64_t)H2_SCAN_BLOCK * H2_SCAN_ITEMS;
        if (X.scan_blocks.ensure((size_t)((p.G + 1 + per_block - 1) / per_block) * 4 + 16)) return 1;
    }
    issue = [&]() -> int {
        if (!p.fast) CU(cudaMemsetAsync(X.counts.p, 0, K * (p.G + 1) * 4, s));
        CU(cudaMemsetAsync(X.cursor.p, 0, K * 2 * p.G * 4, s));
        CU(cudaMemsetAsync(X.size_hist.p, 0, K * small_words * 4, s));
        CU(cudaMemsetAsync(X.bucket_sum.p, 0, K * p.G * sizeof(xyzz), s));
        if (!p.fast) CU(cudaMemsetAsync(X.pkey.p, 0xff, K * part_total * 4, s));

        auto k_bin = msm_bin_kernel<P, PS>;
        auto k_hist = msm_hist_kernel<P, PS>;
        auto k_scatter = msm_scatter_kernel<P, PS>;
        auto k_ihist = msm_item_hist_kernel<P, PS>;
        auto k_ibases = msm_item_bases_kernel<P, PS>;
        auto k_iplace = msm_item_place_kernel<P, PS>;
        auto k_accum0 = msm_accum0_kernel<P, PS>;
        auto k_accum0q = msm_accum0_quad_kernel<P, PS>;
        auto k_accum0p2 = msm_accum0_pair_kernel<P, PS>;
        auto k_accum0s2 = msm_accum0_split_kernel<P, PS, 2>;
        auto k_accum0s4 = msm_accum0_split_kernel<P, PS, 4>;
        auto k_accum0m2 = msm_accum0_multi_kernel<P, PS, 2>;
        auto k_accum0m4 = msm_accum0_multi_kernel<P, PS, 4>;
        auto k_ba = X.ba_variant == 1 ? msm_ba_round_kernel<P, PS, 4, 5> : X.ba_variant == 2 ? msm_ba_round_kernel<P, PS, 2, 4>
                  : X.ba_variant == 3 ? msm_ba_round_kernel<P, PS, 2, 5> : msm_ba_round_kernel<P, PS, 4, 4>;
        auto k_accum0p = msm_accum0_pts_kernel<P, PS>;
        auto k_accumN = msm_accumN_kernel<P, PS>;
        auto k_rest = msm_accum_rest_kernel<P, PS>;
        auto k_reduceA = msm_reduceA_kernel<P, PS>;
        auto k_r0 = msm_r0_kernel<P, PS>;
        auto k_r1 = msm_r1_kernel<P, PS>;
        auto k_wsum = msm_wsum_kernel<P, PS>;
        auto k_final = msm_final_kernel<P, PS>;
        for (uint32_t j = 0; j < K; j++) {
            const MsmPlan &q = pk[j];
            const MsmBuffers &M = Mk[j];
            if (bc && bc->k) {   // the scalars of this chunk (K == 1: of every chunk of the upload)
                for (uint32_t e = (K > 1 ? j : 0); e < (K > 1 ? j + 1 : bc->k); e++) {
                    if (bc->wait_recorded(2 * e + 1)) return fail("msm: the upload of the inputs failed");
                    CU(cudaStreamWaitEvent(s, bc->ev_scal[e], 0));
                }
            }
            // K2/K3: the (point, window) references sorted by bucket -- a single pass into per-bucket bins; the exact
            // histogram / scan / scatter kernels run only if a bin overflowed (flags[1], set by the bin kernel) or if there
            // are no bins (set here)
            if (q.cap == 0) CU(cudaMemsetAsync(M.flags + 1, 0x01, 4, s));
            else LAUNCH(k_bin, blocks_for(q.n * q.sets, 256), 256, 0, s, q, M);
            if (!q.fast) {
                LAUNCH(k_hist, blocks_for(q.n * q.sets, 256), 256, 0, s, q, M);
                if (exclusive_scan_u32(M.counts, q.G + 1, s, M.flags + 1)) return 1;
                LAUNCH(k_scatter, blocks_for(q.n * q.sets, 256), 256, 0, s, q, M);
            }
            // K4: work items (one per bucket, oversized buckets split), largest first
            if (!q.natural) {
                LAUNCH(k_ihist, blocks_for(q.G, 256), 256, 0, s, q, M);
                LAUNCH(k_ibases, 1, 32, 0, s, q, M);
                LAUNCH(k_iplace, blocks_for(q.G, 256), 256, 0, s, q, M);
            }
            if (bc && bc->k) {   // the sort above only needed the scalars
                for (uint32_t e = (K > 1 ? j : 0); e < (K > 1 ? j + 1 : bc->k); e++) {
                    if (bc->wait_recorded(2 * e + 2)) return fail("msm: the upload of the inputs failed");
                    CU(cudaStreamWaitEvent(s, bc->ev[e], 0));
                }
            }
            if (q.glv) {
                auto k_phi = msm_phi_kernel<P, PS>;
                LAUNCH(k_phi, blocks_for(q.n, 256), 256, 0, s, M.bases, M.bases_phi, (uint64_t)q.n);
            }
            prof_begin(PROF_MSM_ACCUM0, s);
            if (q.max_refs <= (q.fixed ? 2 : 1) * H2_MSM_QUAD_ACCUM_REFS) {   // latency-bound: cooperating lanes per work item
                if (X.accum_ways == 4) LAUNCH(k_accum0m4, blocks_for(q.max_items * 16, 128), 128, 0, s, q, M);
                else if (X.accum_ways == 2) LAUNCH(k_accum0m2, blocks_for(q.max_items * 8, 128), 128, 0, s, q, M);
                else if (X.accum_ways == 0) LAUNCH(k_accum0p2, blocks_for(q.max_items * 2, 128), 128, 0, s, q, M);
                else if (X.accum_ways == 12) LAUNCH(k_accum0s2, blocks_for(q.max_items * 2, 128), 128, 0, s, q, M);
                else if (X.accum_ways == 14) LAUNCH(k_accum0s4, blocks_for(q.max_items * 4, 128), 128, 0, s, q, M);
                else LAUNCH(k_accum0q, blocks_for(q.max_items * 4, 128), 128, 0, s, q, M);
            }
            else {
                // batched-affine halving rounds, then the chain over the last level; all of them return at once if the
                // exact sort ran (flags[1]) -- then the classic kernel below does the work, otherwise IT returns at once
                for (uint32_t r = 1; r <= q.ba; r++)
                    LAUNCH(k_ba, blocks_for((q.max_items + q.ba_m[r - 1] - 1) / q.ba_m[r - 1], 128), 128, 0, s, q, M, r);
                if (q.ba) LAUNCH(k_accum0p, blocks_for(q.max_items, 128), 128, 0, s, q, M);
                LAUNCH(k_accum0, blocks_for(q.max_items, 128), 128, 0, s, q, M);
            }
            prof_end(s);
            if (!q.fast) {
                if (q.acc_levels > 1) LAUNCH(k_accumN, blocks_for(q.acc_threads[1], 128), 128, 0, s, q, M, 1u);
                if (q.acc_levels > 2) LAUNCH(k_accumN, blocks_for(q.acc_threads[2], 128), 128, 0, s, q, M, 2u);
                if (q.acc_levels > 3) LAUNCH(k_rest, 1, 256, 0, s, q, M);
            }
        }
        // K5: bucket reduce (adds the per-chunk bucket sums) and window combine
        const MsmBuffers &M = Mk[0];
        LAUNCH(k_reduceA, blocks_for((uint64_t)p.Wb * p.m1 * 4, 128), 128, 0, s, p, M);                    // quads
        LAUNCH(k_r0, blocks_for((uint64_t)p.Wb * p.nb0 * (2 + p.bits0) * 4, 128), 128, 0, s, p, M);
        LAUNCH(k_r1, p.Wb * p.r1_rows, 4 * H2_R1_QUADS, 0, s, p, M);
        LAUNCH(k_wsum, p.Wb, 128, 0, s, p, M);
        LAUNCH(k_final, 1, 64, 0, s, p, M, (uint32_t)out_canonical);
        return 0;
    };
    return msm_issue_or_replay(issue, fixed && !bc, d_scalars, d_bases, d_out, n, stride, c, sets, scalars_mont, out_canonical, fast, s);
}

static int msm_dispatch(int curve, const fe *d_scalars, int scalars_mont, const PassBases &B, size_t n, jacobian *d_out, int out_canonical,
                        cudaStream_t s, const BasesChunks *bc, uint32_t sets, bool fast = false, bool rerun = false, bool *ran_fast = nullptr) {
    return by_curve(curve, [&](auto p, auto ps) {
        return msm_run<decltype(p), decltype(ps)>(d_scalars, scalars_mont, B.bases, n, B.c, B.mode, B.stride, d_out, out_canonical, s, bc, sets,
                                                  fast, rerun, ran_fast);
    });
}

// Where the result of an msm_pass goes: `sets` Jacobian points to host memory, or (affine) as many affine points after
// batch_normalize on the device, or one Jacobian point to `peer` on device `peer_dev` (a multi-GPU worker's partial sum).
struct PassOut { void *host; bool affine = false; void *peer = nullptr; int peer_dev = -1; };
// One MSM pass whose result leaves the device, on the context's stream: issued, normalised (to.affine), copied out and the
// stream synchronised.  A pass over a window table runs fast first (MsmPlan::fast) unless fast passes are off
// (h2_test_set_fast_fixed) or its bases arrive in chunks; if either device flag comes back set -- a bin overflowed or a bucket
// was split -- its result is not valid and the pass runs again, in full.  `issued`, if given, runs after each issue with the
// issue's return code and returns the code to go on with.
static int msm_pass(int curve, const fe *d_scalars, int scalars_mont, const PassBases &B, size_t n, uint32_t sets, jacobian *d_result,
                    int canon, const PassOut &to, const BasesChunks *bc = nullptr, const std::function<int(int)> &issued = nullptr) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (to.affine && X.ec_out.ensure(sets * sizeof(affine))) return 1;
    for (int attempt = 0; attempt < 2; attempt++) {
        bool fast = false;
        int rc = msm_dispatch(curve, d_scalars, scalars_mont, B, n, d_result, to.affine ? 0 : canon, s, bc, sets,
                              attempt == 0 && B.mode == 1 && X.fast_on && !bc, attempt == 1, &fast);
        if (issued) rc = issued(rc);
        if (rc) return rc;
        if (to.affine) {
            const uint32_t nb = blocks_for((sets + H2_NORM_CHUNK - 1) / H2_NORM_CHUNK, 64);
            auto normalize = [&](auto p, auto) {
                LAUNCH(normalize_kernel<decltype(p)>, nb, 64, 0, s, (const xyzz *)nullptr, d_result, 0, X.ec_out.as<affine>(), canon, (uint64_t)sets);
                return 0;
            };
            if (by_curve(curve, normalize)) return 1;
            CU(cudaMemcpyAsync(to.host, X.ec_out.p, sets * sizeof(affine), cudaMemcpyDeviceToHost, s));
        } else if (to.peer) {
            CU(cudaMemcpyPeerAsync(to.peer, to.peer_dev, d_result, X.device, sets * sizeof(jacobian), s));
        } else {
            CU(cudaMemcpyAsync(to.host, d_result, sets * sizeof(jacobian), cudaMemcpyDeviceToHost, s));
        }
        if (fast) {
            if (!X.h_flags) CU(cudaHostAlloc((void **)&X.h_flags, 2 * sizeof(uint32_t), cudaHostAllocDefault));
            CU(cudaMemcpyAsync(X.h_flags, X.last_flags, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        }
        CU(cudaStreamSynchronize(s));
        if (!fast || (X.h_flags[0] == 0 && X.h_flags[1] == 0)) break;
    }
    return 0;
}
// window size for a precomputed table over n bases: few references per bucket (short serial chains)
// for small n, fewer windows for large n
static uint32_t table_window(size_t n) {
    uint32_t lg = 0;
    while ((1ull << (lg + 1)) <= n) lg++;
    // candidates are the window sizes whose TOP window is well filled (scalars have 254 significant bits:
    // 254 - (W - 1) c = 6, 14, 14, 16, 14 bits for c = 8, 15, 16, 17, 20): a top window of 1-2 bits would send n / 4
    // references to a handful of shared buckets and defeat the single-pass sort
    uint32_t want = lg + 2;
    if (want <= 9) return 8;
    if (want <= 15) return 15;
    if (want == 16) return 15;        // k = 14 (tools/table_sweep.py times the IPA opening and commits by window)
    if (want <= 18) return 16;        // k = 15, 16: top window 14 bits
    if (want <= 20) return 17;        // k = 17, 18
    return 20;
}
static int build_table(BaseSet *b, uint32_t c, cudaStream_t s) {
    if (c == 0) c = table_window(b->n);
    if (c < 4 || c > 24) return fail("window table: window bits must be in [4, 24]");
    uint32_t W = (256 + c - 1) / c;
    if ((uint64_t)W * b->n >= (1ull << 31)) return fail("window table: too many points");
    if (b->table.ensure((size_t)W * b->n * sizeof(affine))) return 1;
    if (by_curve(b->curve, [&](auto p, auto ps) {
            auto k = msm_table_kernel<decltype(p), decltype(ps)>;
            LAUNCH(k, blocks_for(b->n, 128), 128, 0, s, b->buf.as<affine>(), b->table.as<affine>(), (uint64_t)b->n, (uint64_t)b->n, c, W);
            return 0;
        }))
        return 1;
    b->c = c; b->W = W;
    return 0;
}
// digit-multiples table of a small resident set (fixedbase.cuh), from the c = 8 window table
#define H2_FB_MAX_POINTS ((1u << 15) + 2u)
static int build_direct(BaseSet *b, cudaStream_t s) {
    if (b->n > H2_FB_MAX_POINTS) return fail("H2_BASES_DIRECT: at most 2^15 + 2 points (256 KiB of table per point)");
    if (b->c != H2_FB_BITS || b->W != H2_FB_WINDOWS) return fail("H2_BASES_DIRECT: needs the 8-bit window table");
    if (b->dtable.ensure((size_t)H2_FB_WINDOWS * H2_FB_MULTIPLES * b->n * sizeof(affine))) return 1;
    const uint64_t threads = (uint64_t)H2_FB_WINDOWS * b->n;
    return by_curve(b->curve, [&](auto p, auto ps) {
        auto k = fb_table_kernel<decltype(p), decltype(ps)>;
        LAUNCH(k, blocks_for(threads, 128), 128, 0, s, (const affine *)b->table.as<affine>(), b->dtable.as<affine>(), (uint64_t)b->n, (uint64_t)b->n);
        return 0;
    });
}
int convert_points(int curve, affine *d, size_t n, int to_mont, cudaStream_t s) {
    return by_curve(curve, [&](auto p, auto) {
        if (n) LAUNCH(convert_points_kernel<decltype(p)>, blocks_for(n, 256), 256, 0, s, d, (uint64_t)n, to_mont);
        return 0;
    });
}

extern "C" int h2_msm_dev(int curve, const void *d_scalars, int scalars_repr, const void *d_bases, size_t n, uint32_t window_bits,
                          void *d_out_xyz, void *stream) {
    CtxLock lk;
    const HostArgs h("h2_msm_dev", scalars_repr);
    if (require_ready() || h.check()) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    StreamSplice splice(s);   // the MSM scratch is the context's
    if (splice.failed) return 1;
    return msm_dispatch(curve, (const fe *)d_scalars, h.mont(), PassBases{(const affine *)d_bases, window_bits}, n, (jacobian *)d_out_xyz, 0, s,
                        nullptr, 1);
}

// host_bases != nullptr: one-shot MSM -- the bases are uploaded (and converted) on the copy stream AFTER the
// scalars, overlapping the digit/sort kernels, which only read scalars (B.bases is where they go).
static int msm_host_common(int curve, const void *scalars, size_t n_scalars, const void *extra_scalar, const PassBases &B,
                           size_t n_total, const HostArgs &h, const PassOut &to, const void *host_bases = nullptr) {
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (X.scal_in.ensure((n_total + 1) * sizeof(fe)) || X.result.ensure(sizeof(jacobian))) return 1;
    BasesChunks bc;
    std::atomic<uint32_t> recorded{0};
    std::atomic<int> up_failed{0};
    std::string up_err;
    std::thread uploader;
    if (host_bases && n_total) {
        // One-shot MSM: everything goes up on the copy stream, interleaved per chunk -- scalars of chunk j, then its
        // bases -- so that the sort of chunk j starts when its scalars have landed and its accumulation when its bases
        // have, while chunk j + 1 is on the link.
        // (2 chunks from 2^chunk_min_log points, 3 from 2x that, 4 from 8x: every chunk pays its own sort / work-item launches)
        cudaStream_t cs = X.copy_stream;
        CU(cudaEventRecord(X.ev_scalars_up, s));
        CU(cudaStreamWaitEvent(cs, X.ev_scalars_up, 0));      // after the prior users of the scratch buffers
        bc.k = 1;
        if (n_total >= ((size_t)1 << X.chunk_min_log) && n_total >= 16 * H2_MAX_UPLOAD_CHUNKS)
            bc.k = n_total >= ((size_t)8 << X.chunk_min_log) ? H2_MAX_UPLOAD_CHUNKS : n_total >= ((size_t)2 << X.chunk_min_log) ? 3u : 2u;
        affine *db = const_cast<affine *>(B.bases);
        for (uint32_t j = 0; j < bc.k; j++) { bc.ev_scal[j] = X.ev_scal_up[j]; bc.ev[j] = X.ev_bases_up[j]; }
        bc.recorded = &recorded; bc.failed = &up_failed;
        Context *ctx = &X;
        const uint32_t k = bc.k;
        // The uploads run on their own host thread: from pageable caller memory they are staged through the pinned ring
        // (upload_async blocks while it copies), and the kernels of chunk j must be issued while chunk j + 1 is staged.
        auto upload = [=, &recorded, &up_failed, &up_err]() {
            set_cur(ctx);
            auto run = [&]() -> int {
                CU(cudaSetDevice(ctx->device));
                for (uint32_t j = 0; j < k; j++) {
                    size_t lo = chunk_first(n_total, k, j), hi = chunk_first(n_total, k, j + 1);
                    if (upload_async(ctx->scal_in.as<fe>() + lo, (const fe *)scalars + lo, (hi - lo) * sizeof(fe), cs)) return 1;
                    CU(cudaEventRecord(ctx->ev_scal_up[j], cs));
                    recorded.store(2 * j + 1, std::memory_order_release);
                    if (upload_async(db + lo, (const affine *)host_bases + lo, (hi - lo) * sizeof(affine), cs)) return 1;
                    if (h.canon() && convert_points(curve, db + lo, hi - lo, 1, cs)) return 1;
                    CU(cudaEventRecord(ctx->ev_bases_up[j], cs));
                    recorded.store(2 * j + 2, std::memory_order_release);
                }
                return 0;
            };
            if (run()) { up_err = last_error_string(); up_failed.store(1); }
        };
        if (n_total * sizeof(affine) >= (4u << 20)) uploader = std::thread(upload);
        else upload();                                        // small: not worth a thread
    } else {
        if (n_scalars && upload_async(X.scal_in.p, scalars, n_scalars * sizeof(fe), s)) return 1;
        if (extra_scalar) CU(cudaMemcpyAsync(X.scal_in.as<fe>() + n_scalars, extra_scalar, sizeof(fe), cudaMemcpyHostToDevice, s));
    }
    auto joined = [&](int rc) -> int {   // the upload's failure is the one to report
        if (uploader.joinable()) uploader.join();
        if (up_failed.load()) { cudaStreamSynchronize(s); cudaStreamSynchronize(X.copy_stream); return fail(up_err); }
        return rc;
    };
    return msm_pass(curve, X.scal_in.as<fe>(), h.mont(), B, n_total, 1, X.result.as<jacobian>(), h.canon(), to,
                    bc.k ? &bc : nullptr, joined);
}

extern "C" int h2_msm(int curve, const void *scalars, const void *bases_xy, size_t n, int repr, void *out_xyz) {
    CtxLock lk;
    const HostArgs h("h2_msm", repr);
    if (require_ready() || check_curve(curve) || h.check({{scalars, "scalars", n != 0}, {bases_xy, "bases_xy", n != 0}, {out_xyz, "out_xyz"}})) return 1;
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (X.bases_in.ensure((n + 1) * sizeof(affine))) return 1;
    return msm_host_common(curve, scalars, n, nullptr, {X.bases_in.as<affine>()}, n, h, {out_xyz}, bases_xy);
}

static int bases_register_impl(int curve, const void *bases_xy, size_t n, const HostArgs &h, uint32_t window_bits, uint32_t flags, uint64_t *handle);
extern "C" int h2_bases_register(int curve, const void *bases_xy, size_t n, int repr, uint64_t *handle) {
    return bases_register_impl(curve, bases_xy, n, {"h2_bases_register", repr}, 0, 0, handle);
}
extern "C" int h2_bases_register_ex(int curve, const void *bases_xy, size_t n, int repr, uint32_t window_bits, uint32_t flags, uint64_t *handle) {
    return bases_register_impl(curve, bases_xy, n, {"h2_bases_register_ex", repr}, window_bits, flags, handle);
}
static int bases_register_impl(int curve, const void *bases_xy, size_t n, const HostArgs &h, uint32_t window_bits, uint32_t flags, uint64_t *handle) {
    CtxLock lk;
    if (require_ready() || check_curve(curve) || h.check({{bases_xy, "bases_xy", n != 0}})) return 1;
    BaseSet *b = new BaseSet();
    b->curve = curve; b->n = n;
    if (b->buf.ensure((n + 1) * sizeof(affine))) { delete b; return 1; }
    cudaStream_t s = g_ctx.stream;
    auto drop = [&]() { cudaStreamSynchronize(s); b->buf.release(); b->table.release(); b->dtable.release(); delete b; return 1; };
    if (n && upload_async(b->buf.p, bases_xy, n * sizeof(affine), s)) return drop();
    if (h.canon() && convert_points(curve, b->buf.as<affine>(), n, 1, s)) return drop();
    const bool direct = (flags & H2_BASES_DIRECT) && (flags & H2_BASES_PRECOMPUTE) && n > 0;
    if ((flags & H2_BASES_PRECOMPUTE) && n > 0 && build_table(b, direct ? H2_FB_BITS : window_bits, s)) return drop();
    if (direct && build_direct(b, s)) return drop();
    if (cudaStreamSynchronize(s) != cudaSuccess) { fail("h2_bases_register: device error while building the tables"); return drop(); }
    const uint64_t id = new_handle();
    {   // shared by every lane from here on (h2_bases_release: capi_core.cu)
        std::lock_guard<std::mutex> reg(g_reg_mu);
        g_bases[id] = b;
    }
    *handle = id;
    return 0;
}
extern "C" int h2_msm_registered(uint64_t handle, const void *scalars, size_t n, const void *extra_scalar, int repr, void *out_xyz) {
    CtxLock lk;
    const HostArgs h("h2_msm_registered", repr);
    if (require_ready() || h.check({{scalars, "scalars", n != 0}, {out_xyz, "out_xyz"}})) return 1;
    BasesRef ref(handle);
    if (!ref.b) return fail("h2_msm_registered: unknown handle");
    BaseSet *b = ref.b;
    size_t total = n + (extra_scalar ? 1 : 0);
    if (total > b->n) return fail("h2_msm_registered: more scalars than registered bases");
    return msm_host_common(b->curve, scalars, n, extra_scalar, pass_bases(b), total, h, {out_xyz});
}

// `batch` scalar vectors of n entries (+ one extra scalar each, the blinds) against a registered base set with a
// window table: one pass, one bucket set per vector.
static int msm_registered_batch_impl(uint64_t handle, const void *scalars, size_t n, const void *extra_scalars, size_t batch, int repr,
                                     void *out, int affine_out);
extern "C" int h2_msm_registered_batch(uint64_t handle, const void *scalars, size_t n, const void *extra_scalars, size_t batch, int repr,
                                       void *out_xyz) {
    return msm_registered_batch_impl(handle, scalars, n, extra_scalars, batch, repr, out_xyz, 0);
}
// the same pass followed by batch_normalize on the device (plonk/prover.rs:305-311: commit every column, then
// C::Curve::batch_normalize): `batch` affine points (64 B) come back instead of Jacobian ones
extern "C" int h2_msm_registered_batch_affine(uint64_t handle, const void *scalars, size_t n, const void *extra_scalars, size_t batch, int repr,
                                              void *out_xy) {
    return msm_registered_batch_impl(handle, scalars, n, extra_scalars, batch, repr, out_xy, 1);
}
static int msm_registered_batch_impl(uint64_t handle, const void *scalars, size_t n, const void *extra_scalars, size_t batch, int repr,
                                     void *out_xyz, int affine_out) {
    CtxLock lk;
    const HostArgs h(affine_out ? "h2_msm_registered_batch_affine" : "h2_msm_registered_batch", repr);
    if (require_ready() || h.check({{scalars, "scalars", n * batch != 0}, {out_xyz, affine_out ? "out_xy" : "out_xyz", batch != 0}})) return 1;
    BasesRef ref(handle);
    if (!ref.b) return fail("h2_msm_registered_batch: unknown handle");
    BaseSet *b = ref.b;
    if (!b->table.p) return fail("h2_msm_registered_batch: the base set has no window table (register with H2_BASES_PRECOMPUTE)");
    if (batch == 0) return 0;
    if (batch > 64) return fail("h2_msm_registered_batch: batch > 64");
    size_t total = n + (extra_scalars ? 1 : 0);
    if (total > b->n) return fail("h2_msm_registered_batch: more scalars than registered bases");
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (X.scal_in.ensure(batch * total * sizeof(fe)) || X.result.ensure(batch * sizeof(jacobian))) return 1;
    fe *d = X.scal_in.as<fe>();
    if (!extra_scalars) {
        if (upload_async(d, scalars, batch * n * sizeof(fe), s)) return 1;
    } else {   // interleave: [poly_k (n) | blind_k] per vector
        CU(cudaMemcpy2DAsync(d, total * sizeof(fe), scalars, n * sizeof(fe), n * sizeof(fe), batch, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpy2DAsync(d + n, total * sizeof(fe), extra_scalars, sizeof(fe), sizeof(fe), batch, cudaMemcpyHostToDevice, s));
    }
    return msm_pass(b->curve, d, h.mont(), pass_bases(b), total, (uint32_t)batch, X.result.as<jacobian>(), h.canon(), {out_xyz, affine_out != 0});
}

extern "C" int h2_point_sum(int curve, const void *points_xyz, size_t g, int repr, void *out_xyz) {
    CtxLock lk;
    const HostArgs h("h2_point_sum", repr);
    if (require_ready() || h.check({{points_xyz, "points_xyz", g != 0}, {out_xyz, "out_xyz"}})) return 1;
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (X.misc.ensure((g + 1) * sizeof(jacobian)) || X.result.ensure(sizeof(jacobian))) return 1;
    if (g) CU(cudaMemcpyAsync(X.misc.p, points_xyz, g * sizeof(jacobian), cudaMemcpyHostToDevice, s));
    const int canon = h.canon();
    if (by_curve(curve, [&](auto p, auto) {
            LAUNCH(point_sum_kernel<decltype(p)>, 1, 32, 0, s, X.misc.as<jacobian>(), (uint32_t)g, canon, X.result.as<jacobian>());
            return 0;
        }))
        return 1;
    CU(cudaMemcpyAsync(out_xyz, X.result.p, sizeof(jacobian), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return 0;
}


// device-pointer form (the partial results of an NCCL all-gather stay on the device): Montgomery in, Montgomery out
extern "C" int h2_point_sum_dev(int curve, const void *d_points_xyz, size_t g, void *d_out_xyz, void *stream) {
    CtxLock lk;
    if (require_ready()) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    return by_curve(curve, [&](auto p, auto) {
        LAUNCH(point_sum_kernel<decltype(p)>, 1, 32, 0, s, (const jacobian *)d_points_xyz, (uint32_t)g, 0, (jacobian *)d_out_xyz);
        return 0;
    });
}

// ------------------------------------------------------------------------------------------------
// single-process multi-GPU MSM (SURVEY.md section 8(b) `h2_msm_multi_gpu`, section 8(e)): contiguous shards of the
// (scalar, base) arrays, one worker thread and one full single-GPU pipeline per device, the 96-byte partial results written
// into the primary device's memory over NVLink (peer copy), one G-term sum there.  Results are the same group element
// whatever the number of devices.
// ------------------------------------------------------------------------------------------------
extern std::vector<int> g_multi;
static inline void shard_range(size_t n, size_t g, size_t G, size_t *lo, size_t *hi) {
    const size_t base = n / G, rem = n % G;
    *lo = g * base + (g < rem ? g : rem);
    *hi = *lo + base + (g < rem ? 1 : 0);
}
// runs fn(g) on one thread per device with that device's context current; collects the first error
static int multi_run(const std::function<int(size_t)> &fn) {
    const size_t G = g_multi.size();
    std::vector<std::string> errs(G);
    std::vector<int> rcs(G, 0);
    std::vector<std::thread> th;
    for (size_t g = 0; g < G; g++)
        th.emplace_back([&, g]() {
            set_cur(&g_ctxs[g_multi[g]]);
            if (cudaSetDevice(g_multi[g]) != cudaSuccess) { rcs[g] = 1; errs[g] = "cudaSetDevice failed"; return; }
            rcs[g] = fn(g);
            if (rcs[g]) errs[g] = last_error_string();
        });
    for (auto &t : th) t.join();
    cudaSetDevice(g_primary->device);
    for (size_t g = 0; g < G; g++) if (rcs[g]) return fail("device " + std::to_string(g_multi[g]) + ": " + errs[g]);
    return 0;
}
static int multi_finish(int curve, const HostArgs &h, void *out_xyz) {     // the G-term sum on the primary device
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    const size_t G = g_multi.size();
    const int canon = h.canon();
    if (X.result.ensure(sizeof(jacobian))) return 1;
    if (by_curve(curve, [&](auto p, auto) {
            LAUNCH(point_sum_kernel<decltype(p)>, 1, 32, 0, s, X.multi_parts.as<jacobian>(), (uint32_t)G, canon, X.result.as<jacobian>());
            return 0;
        }))
        return 1;
    CU(cudaMemcpyAsync(out_xyz, X.result.p, sizeof(jacobian), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    return 0;
}
// The h2_multi_* calls run on the primary context: they hold its mutex for the whole call, and g_multi, g_multi_bases and
// the secondary devices' contexts change only under it (and g_reg_mu).  A thread bound to a lane is refused.
static int multi_refuse_lane(const char *who) {
    if (on_lane()) return fail(std::string(who) + ": the multi-GPU entry points run on the primary context, not on a lane (h2_lane_bind(0))");
    return 0;
}
extern "C" int h2_msm_multi_gpu(int curve, const void *scalars, const void *bases_xy, size_t n, int repr, void *out_xyz) {
    if (multi_refuse_lane("h2_msm_multi_gpu")) return 1;
    CtxLock lk;
    const HostArgs h("h2_msm_multi_gpu", repr);
    if (require_ready() || check_curve(curve) || h.check({{scalars, "scalars", n != 0}, {bases_xy, "bases_xy", n != 0}, {out_xyz, "out_xyz"}})) return 1;
    if (g_multi.empty()) return fail("h2_msm_multi_gpu: call h2_multi_init first");
    const size_t G = g_multi.size();
    Context &P0 = *g_primary;
    if (P0.multi_parts.ensure(G * sizeof(jacobian))) return 1;
    jacobian *parts = P0.multi_parts.as<jacobian>();
    const int prim = P0.device;
    int rc = multi_run([&](size_t g) -> int {
        Context &X = g_ctx;
        size_t lo, hi;
        shard_range(n, g, G, &lo, &hi);
        if (X.bases_in.ensure((hi - lo + 1) * sizeof(affine))) return 1;
        return msm_host_common(curve, (const fe *)scalars + lo, hi - lo, nullptr, {X.bases_in.as<affine>()}, hi - lo, h,
                               {nullptr, false, parts + g, prim}, (const affine *)bases_xy + lo);
    });
    if (rc) return rc;
    return multi_finish(curve, h, out_xyz);
}
// resident shards: bases[lo_g, hi_g) live on device g, in that device context's `shards` (handle valid for
// h2_msm_multi_registered only).  Handles come from new_handle(), so one from before an h2_shutdown is unknown after it.
struct MultiBases { int curve; size_t n; std::vector<uint64_t> handles; };
static std::map<uint64_t, MultiBases> g_multi_bases;
void multi_bases_clear() { g_multi_bases.clear(); }   // h2_shutdown (the shards go with their contexts)
extern "C" int h2_multi_bases_register(int curve, const void *bases_xy, size_t n, int repr, uint64_t *handle) {
    if (multi_refuse_lane("h2_multi_bases_register")) return 1;
    CtxLock lk;
    const HostArgs h("h2_multi_bases_register", repr);
    if (require_ready() || check_curve(curve) || h.check({{bases_xy, "bases_xy", n != 0}})) return 1;
    if (g_multi.empty()) return fail("h2_multi_bases_register: call h2_multi_init first");
    const size_t G = g_multi.size();
    MultiBases mb;
    mb.curve = curve; mb.n = n; mb.handles.assign(G, 0);
    int rc = multi_run([&](size_t g) -> int {
        Context &X = g_ctx;
        size_t lo, hi;
        shard_range(n, g, G, &lo, &hi);
        BaseSet *b = new BaseSet();
        b->curve = curve; b->n = hi - lo;
        if (b->buf.ensure((hi - lo + 1) * sizeof(affine))) { delete b; return 1; }
        cudaStream_t s = X.stream;
        if (upload_async(b->buf.p, (const affine *)bases_xy + lo, (hi - lo) * sizeof(affine), s) ||
            (h.canon() && convert_points(curve, b->buf.as<affine>(), hi - lo, 1, s)) ||
            cudaStreamSynchronize(s) != cudaSuccess) {
            cudaStreamSynchronize(s); b->buf.release(); delete b;
            return fail("h2_multi_bases_register: upload failed");
        }
        mb.handles[g] = new_handle();
        X.shards[mb.handles[g]] = b;
        return 0;
    });
    if (rc) return rc;
    *handle = new_handle();
    std::lock_guard<std::mutex> reg(g_reg_mu);
    g_multi_bases[*handle] = mb;
    return 0;
}
extern "C" int h2_multi_bases_release(uint64_t handle) {
    if (multi_refuse_lane("h2_multi_bases_release")) return 1;
    CtxLock lk;
    MultiBases mb;
    {
        std::lock_guard<std::mutex> reg(g_reg_mu);
        auto it = g_multi_bases.find(handle);
        if (it == g_multi_bases.end()) return fail("h2_multi_bases_release: unknown handle");
        mb = it->second;
        g_multi_bases.erase(it);
    }
    return multi_run([&](size_t g) -> int {
        Context &X = g_ctx;
        auto ib = X.shards.find(mb.handles[g]);
        if (ib == X.shards.end()) return 0;
        cudaDeviceSynchronize();
        ib->second->buf.release(); ib->second->table.release(); ib->second->dtable.release();
        delete ib->second;
        X.shards.erase(ib);
        return 0;
    });
}
extern "C" int h2_msm_multi_registered(uint64_t handle, const void *scalars, size_t n, int repr, void *out_xyz) {
    if (multi_refuse_lane("h2_msm_multi_registered")) return 1;
    CtxLock lk;
    const HostArgs h("h2_msm_multi_registered", repr);
    if (require_ready() || h.check({{scalars, "scalars", n != 0}, {out_xyz, "out_xyz"}})) return 1;
    auto it = g_multi_bases.find(handle);
    if (it == g_multi_bases.end()) return fail("h2_msm_multi_registered: unknown handle");
    const MultiBases &mb = it->second;
    if (n != mb.n) return fail("h2_msm_multi_registered: scalar count differs from the registered bases");
    if (mb.handles.size() != g_multi.size()) return fail("h2_msm_multi_registered: the device set changed since registration");
    const size_t G = g_multi.size();
    Context &P0 = *g_primary;
    if (P0.multi_parts.ensure(G * sizeof(jacobian))) return 1;
    jacobian *parts = P0.multi_parts.as<jacobian>();
    const int prim = P0.device;
    int rc = multi_run([&](size_t g) -> int {
        Context &X = g_ctx;
        size_t lo, hi;
        shard_range(n, g, G, &lo, &hi);
        auto ib = X.shards.find(mb.handles[g]);
        if (ib == X.shards.end()) return fail("h2_msm_multi_registered: a shard was released");
        return msm_host_common(mb.curve, (const fe *)scalars + lo, hi - lo, nullptr, {ib->second->buf.as<affine>()}, hi - lo, h,
                               {nullptr, false, parts + g, prim});
    });
    if (rc) return rc;
    return multi_finish(mb.curve, h, out_xyz);
}

// ------------------------------------------------------------------------------------------------
static void ipa_free(IpaSession *q) {   // back to the pool (the caller has synchronised the stream)
    if (g_ctx.ipa_pool.size() < 2) { g_ctx.ipa_pool.push_back(q); return; }
    q->p.release(); q->b.release(); q->s.release(); q->scal.release(); q->out.release(); delete q;
}
static IpaState ipa_state(IpaSession *q) {
    IpaState S;
    S.p = q->p.as<fe>(); S.b = q->b.as<fe>(); S.s = q->s.as<fe>(); S.scal = q->scal.as<fe>(); S.n = 1ull << q->k;
    return S;
}
template <class PS> static int ipa_begin_impl(IpaSession *q, const void *p_prime, PolyBuf *p_poly, const void *x3, const HostArgs &h, cudaStream_t s) {
    Context &X = g_ctx;
    const uint64_t n = 1ull << q->k;
    if (q->p.ensure(n * sizeof(fe)) || q->b.ensure(n * sizeof(fe)) || q->s.ensure(n * sizeof(fe)) || q->scal.ensure(2 * (n + 2) * sizeof(fe)) ||
        q->out.ensure(2 * sizeof(jacobian)) || X.pow2.ensure(64 * sizeof(fe)))
        return 1;
    if (p_poly) CU(cudaMemcpyAsync(q->p.p, p_poly->buf.p, n * sizeof(fe), cudaMemcpyDeviceToDevice, s));
    else if (upload_async(q->p.p, p_prime, n * sizeof(fe), s)) return 1;
    IpaState S = ipa_state(q);
    LAUNCH(ipa_init_kernel<PS>, blocks_for(n, 256), 256, 0, s, S, p_poly ? 1 : h.mont());
    // b_t = x3^t (prover.rs:86-93) with the NTT twiddle generator
    LAUNCH(twiddle_pow2_kernel<PS>, 1, 32, 0, s, X.pow2.as<fe>(), h.elem<PS>(x3), q->k + 1);
    LAUNCH(twiddle_fill_kernel<PS>, blocks_for((n + 31) / 32, 128), 128, 0, s, S.b, X.pow2.as<fe>(), n);
    return 0;
}
static int ipa_begin_common(uint64_t bases_handle, uint32_t k, const void *p_prime, const uint64_t *p_poly_handle, const void *x3, int repr,
                            uint64_t *session);
extern "C" int h2_ipa_begin(uint64_t bases_handle, uint32_t k, const void *p_prime, const void *x3, int repr, uint64_t *session) {
    return ipa_begin_common(bases_handle, k, p_prime, nullptr, x3, repr, session);
}
// p' taken from a device-resident polynomial (Montgomery form): nothing but x3 goes up
extern "C" int h2_ipa_begin_poly(uint64_t bases_handle, uint32_t k, uint64_t p_prime_poly, const void *x3, int repr, uint64_t *session) {
    return ipa_begin_common(bases_handle, k, nullptr, &p_prime_poly, x3, repr, session);
}
// The session counts as a user of its base set until h2_ipa_finish: h2_bases_release refuses the set meanwhile.
static int ipa_begin_common(uint64_t bases_handle, uint32_t k, const void *p_prime, const uint64_t *p_poly_handle, const void *x3, int repr,
                            uint64_t *session) {
    CtxLock lk;
    const HostArgs h(p_poly_handle ? "h2_ipa_begin_poly" : "h2_ipa_begin", repr);
    if (require_ready() || h.check({{p_prime, "p_prime", !p_poly_handle}, {x3, "x3"}})) return 1;
    BasesRef ref(bases_handle, true);
    if (!ref.b) return fail("h2_ipa_begin: unknown bases handle");
    BaseSet *b = ref.b;
    bool opened = false;
    struct SessionGuard {   // the session count goes back unless the session opens
        const uint64_t h; const bool &opened;
        ~SessionGuard() { if (!opened) bases_session_end(h); }
    } guard{bases_handle, opened};
    if (k == 0 || k > 28) return fail("h2_ipa_begin: k out of range");
    if (b->n != (1ull << k) + 2) return fail("h2_ipa_begin: the base set must hold g[0..2^k) || w || u");
    if (!b->table.p) return fail("h2_ipa_begin: the base set has no window table (register with H2_BASES_PRECOMPUTE)");
    return by_curve(b->curve, [&](auto, auto ps) {
        using PS = decltype(ps);
        PolyArgs g("h2_ipa_begin_poly", PS::ID);
        PolyBuf *p_poly = nullptr;
        if (p_poly_handle && !(p_poly = g.in(*p_poly_handle, "p_prime_poly", 1ull << k, "2^k"))) return 1;   // looked up and used under the one lock
        IpaSession *q;
        if (!g_ctx.ipa_pool.empty()) { q = g_ctx.ipa_pool.back(); g_ctx.ipa_pool.pop_back(); }
        else q = new IpaSession();
        q->bases = bases_handle; q->k = k; q->round = 0; q->folded = 1;
        cudaStream_t s = g_ctx.stream;
        if (ipa_begin_impl<PS>(q, p_prime, p_poly, x3, h, s)) { ipa_free(q); return 1; }
        cudaError_t e = cudaStreamSynchronize(s);   // p_prime may be pageable host memory
        if (e != cudaSuccess) { ipa_free(q); return fail(std::string("h2_ipa_begin: ") + cudaGetErrorString(e)); }
        uint64_t id = new_handle();
        g_ctx.ipa[id] = q;
        *session = id;
        opened = true;
        return 0;
    });
}
static int ipa_round_common(uint64_t session, const void *z, const void *l_rand, const void *r_rand, int repr, void *out, int affine_out);
extern "C" int h2_ipa_round(uint64_t session, const void *z, const void *l_rand, const void *r_rand, int repr, void *out_lr_xyz) {
    return ipa_round_common(session, z, l_rand, r_rand, repr, out_lr_xyz, 0);
}
// L_j, R_j as the two AFFINE points the prover writes to the transcript (prover.rs:120-125 `to_affine`), 2 x 64 B
extern "C" int h2_ipa_round_affine(uint64_t session, const void *z, const void *l_rand, const void *r_rand, int repr, void *out_lr_xy) {
    return ipa_round_common(session, z, l_rand, r_rand, repr, out_lr_xy, 1);
}
static int ipa_round_common(uint64_t session, const void *z, const void *l_rand, const void *r_rand, int repr, void *out_lr_xyz, int affine_out) {
    CtxLock lk;
    const HostArgs h(affine_out ? "h2_ipa_round_affine" : "h2_ipa_round", repr);
    if (require_ready() || h.check({{z, "z"}, {l_rand, "l_rand"}, {r_rand, "r_rand"}, {out_lr_xyz, affine_out ? "out_lr_xy" : "out_lr_xyz"}})) return 1;
    auto it = g_ctx.ipa.find(session);
    if (it == g_ctx.ipa.end()) return fail("h2_ipa_round: unknown session");
    IpaSession *q = it->second;
    BasesRef ref(q->bases);
    if (!ref.b) return fail("h2_ipa_round: the session's base set was released");
    if (q->round >= q->k) return fail("h2_ipa_round: all k rounds are done");
    if (!q->folded) return fail("h2_ipa_round: h2_ipa_fold must follow each round");
    BaseSet *b = ref.b;
    cudaStream_t s = g_ctx.stream;
    const uint64_t n = 1ull << q->k;
    const IpaState S = ipa_state(q);
    // S.scal from p, b and s: a re-run of the pass reads them again, as no MSM kernel writes its scalars
    int rc = by_curve(b->curve, [&](auto, auto ps) {
        using PS = decltype(ps);
        const uint32_t bit = q->k - 1 - q->round;
        LAUNCH(ipa_prep_kernel<PS>, blocks_for(n, 256), 256, 0, s, S, bit);
        LAUNCH(ipa_inner_kernel<PS>, 1, 512, 0, s, S, bit, h.elem<PS>(z), h.elem<PS>(l_rand), h.elem<PS>(r_rand));
        return 0;
    });
    if (rc || msm_pass(b->curve, S.scal, 1, pass_bases(b), n + 2, 2, q->out.as<jacobian>(), h.canon(), {out_lr_xyz, affine_out != 0}))
        return 1;
    q->folded = 0;
    return 0;
}
extern "C" int h2_ipa_fold(uint64_t session, const void *u, const void *u_inv, int repr) {
    CtxLock lk;
    const HostArgs h("h2_ipa_fold", repr);
    if (require_ready() || h.check({{u, "u"}, {u_inv, "u_inv"}})) return 1;
    auto it = g_ctx.ipa.find(session);
    if (it == g_ctx.ipa.end()) return fail("h2_ipa_fold: unknown session");
    IpaSession *q = it->second;
    BasesRef ref(q->bases);
    if (!ref.b) return fail("h2_ipa_fold: the session's base set was released");
    if (q->folded) return fail("h2_ipa_fold: no round to fold");
    const uint64_t n = 1ull << q->k;
    const uint32_t bit = q->k - 1 - q->round;
    cudaStream_t s = g_ctx.stream;
    IpaState S = ipa_state(q);
    if (by_curve(ref.b->curve, [&](auto, auto ps) {
            using PS = decltype(ps);
            LAUNCH(ipa_fold_kernel<PS>, blocks_for(n, 256), 256, 0, s, S, bit, h.elem<PS>(u), h.elem<PS>(u_inv));
            return 0;
        }))
        return 1;
    q->round++; q->folded = 1;   // asynchronous: the next round (or finish) is ordered behind it on the stream
    return 0;
}
// out_c_b == NULL aborts the session whatever repr is, so that cleanup cannot fail
extern "C" int h2_ipa_finish(uint64_t session, int repr, void *out_c_b) {
    CtxLock lk;
    const HostArgs h("h2_ipa_finish", repr);
    if (require_ready() || (out_c_b && h.check())) return 1;
    auto it = g_ctx.ipa.find(session);
    if (it == g_ctx.ipa.end()) return fail("h2_ipa_finish: unknown session");
    IpaSession *q = it->second;
    int rc = 0;
    cudaStream_t s = g_ctx.stream;
    BasesRef ref(q->bases);
    if (out_c_b) {
        if (!ref.b) rc = fail("h2_ipa_finish: the session's base set was released");
        else if (q->round != q->k || !q->folded) rc = fail("h2_ipa_finish: the k rounds are not complete");
        else {
            IpaState S = ipa_state(q);
            fe *out = q->scal.as<fe>();
            rc = by_curve(ref.b->curve, [&](auto, auto ps) {
                ipa_result_kernel<decltype(ps)><<<1, 32, 0, s>>>(S, h.canon(), out);
                g_launches.fetch_add(1, std::memory_order_relaxed);
                cudaError_t e = cudaMemcpyAsync(out_c_b, out, 2 * sizeof(fe), cudaMemcpyDeviceToHost, s);
                return e != cudaSuccess ? fail(std::string("h2_ipa_finish: ") + cudaGetErrorString(e)) : 0;
            });
        }
    }
    cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess && !rc) rc = fail(std::string("h2_ipa_finish: ") + cudaGetErrorString(e));
    bases_session_end(q->bases);
    ipa_free(q);
    g_ctx.ipa.erase(it);
    return rc;
}


// commit(poly, blind) = <poly[0..n), bases[0..n)> + blind * bases[n] for `batch` resident polynomials in one pass
static int msm_registered_polys_impl(uint64_t bases_handle, const uint64_t *polys, size_t batch, size_t n, const void *extra_scalars, int repr,
                                     void *out_xyz, int affine_out);
extern "C" int h2_msm_registered_polys(uint64_t bases_handle, const uint64_t *polys, size_t batch, size_t n, const void *extra_scalars, int repr,
                                       void *out_xyz) {
    return msm_registered_polys_impl(bases_handle, polys, batch, n, extra_scalars, repr, out_xyz, 0);
}
// ... followed by batch_normalize on the device: `batch` affine points (64 B), what the prover writes to the transcript
extern "C" int h2_msm_registered_polys_affine(uint64_t bases_handle, const uint64_t *polys, size_t batch, size_t n, const void *extra_scalars,
                                              int repr, void *out_xy) {
    return msm_registered_polys_impl(bases_handle, polys, batch, n, extra_scalars, repr, out_xy, 1);
}
static int msm_registered_polys_impl(uint64_t bases_handle, const uint64_t *polys, size_t batch, size_t n, const void *extra_scalars, int repr,
                                     void *out_xyz, int affine_out) {
    CtxLock lk;
    const HostArgs h(affine_out ? "h2_msm_registered_polys_affine" : "h2_msm_registered_polys", repr);
    if (require_ready() || h.check({{out_xyz, affine_out ? "out_xy" : "out_xyz", batch != 0}})) return 1;
    BasesRef ref(bases_handle);
    if (!ref.b) return fail("h2_msm_registered_polys: unknown bases handle");
    BaseSet *b = ref.b;
    if (batch == 0) return 0;
    if (batch > 64) return fail("h2_msm_registered_polys: batch > 64");
    if (batch > 1 && !b->table.p) return fail("h2_msm_registered_polys: a batch needs a base set with a window table (H2_BASES_PRECOMPUTE)");
    const size_t total = n + (extra_scalars ? 1 : 0);
    if (total > b->n) return fail("h2_msm_registered_polys: more scalars than registered bases");
    return by_curve(b->curve, [&](auto, auto ps) {
        PolyArgs g("h2_msm_registered_polys", decltype(ps)::ID);
        std::vector<PolyBuf *> q;
        if (g.in(polys, batch, "polys", n, "n", q)) return 1;
        Context &X = g_ctx;
        cudaStream_t s = X.stream;
        if (X.scal_in.ensure(batch * total * sizeof(fe)) || X.result.ensure(batch * sizeof(jacobian)) || X.misc.ensure(batch * sizeof(fe) + 64)) return 1;
        fe *d = X.scal_in.as<fe>();
        if (extra_scalars && h.up(decltype(ps)::ID, X.misc.as<fe>(), extra_scalars, batch, s)) return 1;   // the blinds: Montgomery form like the resident data
        for (size_t j = 0; j < batch; j++) {
            CU(cudaMemcpyAsync(d + j * total, q[j]->buf.p, n * sizeof(fe), cudaMemcpyDeviceToDevice, s));
            if (extra_scalars) CU(cudaMemcpyAsync(d + j * total + n, X.misc.as<fe>() + j, sizeof(fe), cudaMemcpyDeviceToDevice, s));
        }
        return msm_pass(b->curve, d, 1, pass_bases(b), total, (uint32_t)batch, X.result.as<jacobian>(), h.canon(), {out_xyz, affine_out != 0});
    });
}

