// TEST-ONLY serial execution of the polynomial reductions (polyops.cuh) on the chunk trees of gp_reduce_plan and
// gp_scan_plan, as capi_poly.cu's polyops_run and grand_product_run run them.
#include <cstring>
#include <vector>
#include "polyops.cuh"
using namespace h2;

// mode 0: eval, 1: inner product, 2: kate division.  a, c: batch x n canonical; points: batch canonical; out: eval / inner ->
// batch x 32, kate -> batch x (n - 1) x 32.
template <class P> static int run_polyops(int mode, const uint8_t *a_in, const uint8_t *c_in, uint32_t batch, uint64_t n, const uint8_t *points, uint8_t *out) {
    std::vector<std::vector<fe>> a(batch, std::vector<fe>(n)), c(batch, std::vector<fe>(n));
    std::vector<const fe *> ap(batch), cp(batch);
    std::vector<fe *> qp(batch);
    for (uint32_t b = 0; b < batch; b++) {
        for (uint64_t i = 0; i < n; i++) {
            memcpy(a[b][i].v, a_in + 32 * (b * n + i), 32); a[b][i] = fe_to_mont<P>(a[b][i]);
            if (c_in) { memcpy(c[b][i].v, c_in + 32 * (b * n + i), 32); c[b][i] = fe_to_mont<P>(c[b][i]); }
        }
        ap[b] = a[b].data(); cp[b] = c[b].data(); qp[b] = c[b].data();
    }
    GpTree T;
    if (gp_reduce_plan(n, batch, mode == 1, &T)) return -1;
    const uint64_t *m = T.m, *off = T.off;
    const size_t L = T.L;
    std::vector<fe> lvl(T.total), qarr(T.total), pts((L + 2) * batch);
    for (uint32_t b = 0; b < batch; b++) {
        if (mode == 1) pts[b] = fe_one<P>();
        else { memcpy(pts[b].v, points + 32 * b, 32); pts[b] = fe_to_mont<P>(pts[b]); }
    }
    for (size_t l = 0; l < L; l++) {
        for (uint32_t b = 0; b < batch; b++)
            for (uint64_t t = 0; t < m[l + 1]; t++) {
                if (l == 0 && mode == 1) PolyOps<P>::inner_level0_body(ap.data(), cp.data(), m[0], lvl.data() + off[1], m[1], b, t);
                else PolyOps<P>::eval_level_body(l == 0 ? ap.data() : nullptr, l == 0 ? nullptr : lvl.data() + off[l], m[l], pts.data() + l * batch,
                                                 lvl.data() + off[l + 1], m[l + 1], b, t);
            }
        for (uint32_t b = 0; b < batch; b++) {
            if (mode != 1) PolyOps<P>::pow_chunk_body(pts.data() + l * batch, pts.data() + (l + 1) * batch, b);
            else pts[(l + 1) * batch + b] = fe_one<P>();
        }
    }
    if (mode != 2) {
        for (uint32_t b = 0; b < batch; b++) {
            fe r = L == 0 ? a[b][0] : lvl[off[L] + b];
            r = fe_from_mont<P>(r);
            memcpy(out + 32 * b, r.v, 32);
        }
        return (int)L;
    }
    for (size_t l = L; l-- > 0;) {
        const fe *carry = (l + 1 < L) ? qarr.data() + off[l + 1] : nullptr;
        for (uint32_t b = 0; b < batch; b++)
            for (uint64_t t = 0; t < m[l + 1]; t++)
                PolyOps<P>::kate_down_body(l == 0 ? ap.data() : nullptr, l == 0 ? nullptr : lvl.data() + off[l], m[l], pts.data() + l * batch, carry, m[l + 1],
                                           l == 0 ? nullptr : qarr.data() + off[l], l == 0 ? qp.data() : nullptr, b, t);
    }
    for (uint32_t b = 0; b < batch; b++)
        for (uint64_t i = 0; i + 1 < n; i++) { fe r = fe_from_mont<P>(c[b][i]); memcpy(out + 32 * (b * (n - 1) + i), r.v, 32); }
    return (int)L;
}
extern "C" int emu_polyops(int field, int mode, const uint8_t *a, const uint8_t *c, uint32_t batch, uint64_t n, const uint8_t *points, uint8_t *out) {
    return field == 0 ? run_polyops<FpParams>(mode, a, c, batch, n, points, out) : run_polyops<FqParams>(mode, a, c, batch, n, points, out);
}

// batch_invert in place (mode 0) / exclusive running product with `init` (mode 1: out[0] = init, out[i] = out[i-1] * a[i-1]), with
// the chunk tree of gp_scan_plan.  a: n canonical elements.
template <class P> static int run_grand(int mode, const uint8_t *a_in, uint64_t n, const uint8_t *init, uint8_t *out) {
    std::vector<fe> a(n);
    for (uint64_t i = 0; i < n; i++) { memcpy(a[i].v, a_in + 32 * i, 32); a[i] = fe_to_mont<P>(a[i]); }
    if (mode == 0) {
        for (uint64_t t = 0; t * 16 < n; t++) GrandProduct<P>::invert_body(a.data(), n, t);
        for (uint64_t i = 0; i < n; i++) { fe r = fe_from_mont<P>(a[i]); memcpy(out + 32 * i, r.v, 32); }
        return 0;
    }
    fe in0; memcpy(in0.v, init, 32); in0 = fe_to_mont<P>(in0);
    GpTree T;
    if (gp_scan_plan(n, 1, false, &T)) return -1;
    const uint64_t *m = T.m, *off = T.off;
    const size_t L = T.L;
    std::vector<fe> lvl(T.total), ex(T.total), o(n);
    for (size_t l = 0; l < L; l++)
        for (uint64_t t = 0; t < m[l + 1]; t++) GrandProduct<P>::up_body(l == 0 ? a.data() : lvl.data() + off[l], m[l], lvl.data() + off[l + 1], m[l + 1], t);
    for (size_t l = L + 1; l-- > 0;) {
        const uint64_t chunks = (m[l] + H2_POLY_CHUNK - 1) / H2_POLY_CHUNK;
        const fe *carry = l == L ? nullptr : ex.data() + off[l + 1];
        for (uint64_t t = 0; t < chunks; t++)
            GrandProduct<P>::down_body(l == 0 ? a.data() : lvl.data() + off[l], m[l], carry, in0, l == 0 ? o.data() : ex.data() + off[l], chunks, t);
    }
    for (uint64_t i = 0; i < n; i++) { fe r = fe_from_mont<P>(o[i]); memcpy(out + 32 * i, r.v, 32); }
    return (int)L;
}
extern "C" int emu_grand_product(int field, int mode, const uint8_t *a, uint64_t n, const uint8_t *init, uint8_t *out) {
    return field == 0 ? run_grand<FpParams>(mode, a, n, init, out) : run_grand<FqParams>(mode, a, n, init, out);
}

// The chunk-tree plans themselves.  rule 0: gp_reduce_plan, 1: the same for an inner product, 2: gp_scan_plan, 3: the same
// with level 1.  m, off: H2_GP_MAX_LEVELS values each.  Returns 1 when the plan refuses n.
extern "C" int emu_chunk_tree(int rule, uint64_t n, uint64_t batch, uint64_t *m, uint64_t *off, uint32_t *L, uint64_t *total) {
    GpTree T;
    if (rule < 2 ? gp_reduce_plan(n, batch, rule == 1, &T) : gp_scan_plan(n, batch, rule == 3, &T)) return 1;
    memcpy(m, T.m, sizeof T.m);
    memcpy(off, T.off, sizeof T.off);
    *L = T.L;
    *total = T.total;
    return 0;
}
