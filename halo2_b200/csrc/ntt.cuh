// NTT kernels (K7/K8/K9 in SURVEY.md section 2.1) for Fp / Fq.
//
// Computes exactly the butterfly NETWORK of best_fft
// (/root/reference/halo2_proofs/src/arithmetic.rs:192-295): bit-reversal, twiddles w^i,
// log_n radix-2 DIT stages with  t = b * tw; b = a - t; a = a + t.  No step assumes
// w^n = 1 (benches/fft.rs:17 passes a random w), so the output is bit-identical to the
// reference for ANY omega.
//
// Data movement.  The data stays at its natural index j through all passes; the network's
// "position" p = bitrev(j) is only materialised by the last pass, which stores out[p].
// Stage s (1-based) pairs positions that differ in bit s-1 of p, i.e. elements that differ
// in bit log_n-s of j, with twiddle exponent (p mod 2^(s-1)) * 2^(log_n-s).
// A pass handles `sp` consecutive stages on a tile of R = 2^sp rows x C = 2^logc columns held
// in shared memory (two uint4 planes, row stride C+1 -> conflict-free for both row-fastest
// and column-fastest access):
//   geometry A (not last pass): rows = the sp bits of j being transformed, columns = C
//       adjacent j (coalesced C*32 B runs); all columns of a tile share their twiddles.
//   geometry B (last pass): rows = the low sp bits of j (contiguous in memory), columns = C
//       blocks whose outputs p are adjacent, so the bit-reversed store is coalesced too.
// Columns: one launch per pass covers every column of a batch (grid.y = column; NttPassArgs::in_cols / out_cols).
// Fusions: first pass can zero-pad (coeff_to_extended's resize, poly/domain.rs:248) and
// multiply element j by in_scale[j mod 3] (distribute_powers_zeta, :357-373, and/or the
// canonical->Montgomery factor); last pass can multiply output p by out_scale[p mod 3]
// (ifft divisor :375-383, coset un-scale :303-325, and/or Montgomery->canonical).
// The vanishing argument's quotient (K24) adds two more: the first pass can multiply element j by in_table[j & in_mask]
// (divide_by_vanishing_poly, :329-348), and the last pass can scatter output p into pieces of 2^piece_log coefficients,
// out_cols[p >> piece_log] + (p mod 2^piece_log) (h_poly.chunks_exact(n), plonk/vanishing/prover.rs:95-100).
#pragma once
#include "field.cuh"

namespace h2 {

enum : uint32_t { NTT_FIRST = 1u, NTT_LAST = 2u, NTT_IN_SCALE = 4u, NTT_OUT_SCALE = 8u, NTT_IN_TABLE = 16u, NTT_OUT_PIECES = 32u };

struct NttPassArgs {
    const fe *in;
    fe *out;
    const fe *tw;        // w^i for i < n/2, Montgomery form
    uint32_t log_n;      // transform size
    uint32_t s0;         // stages completed before this pass
    uint32_t sp;         // stages in this pass
    uint32_t logc;       // log2(columns per tile)
    uint32_t flags;
    uint32_t in_log_n;   // elements with j >= 2^in_log_n read as zero (first pass)
    uint64_t out_len;    // last pass: outputs with p >= out_len are dropped (truncate)
    fe in_scale[3];
    fe out_scale[3];
    // A launch covers gridDim.y columns of one size and domain.  Column c reads in_cols[c] when the table is set, else
    // in + c * in_stride, and writes out_cols[c], else out + c * out_stride.  One column: in / out, no tables.
    const fe *const *in_cols = nullptr;
    fe *const *out_cols = nullptr;
    uint64_t in_stride = 0, out_stride = 0;
    // NTT_IN_TABLE (first pass): element j is multiplied by in_table[j & in_mask] as it is loaded.  NTT_OUT_PIECES (last pass,
    // one column): output p goes to out_cols[p >> piece_log] + (p & (2^piece_log - 1)); out_len drops the tail as usual.
    const fe *in_table = nullptr;
    uint32_t in_mask = 0, piece_log = 0;
};
H2_HD const fe *ntt_col_in(const NttPassArgs &A, uint32_t c) { return A.in_cols ? A.in_cols[c] : A.in + c * A.in_stride; }
H2_HD fe *ntt_col_out(const NttPassArgs &A, uint32_t c) { return A.out_cols ? A.out_cols[c] : A.out + c * A.out_stride; }

H2_HD uint32_t bitrev32(uint32_t x, uint32_t bits) {
    // bits in [0, 32]
    if (bits == 0) return 0;
    x = ((x & 0x55555555u) << 1) | ((x >> 1) & 0x55555555u);
    x = ((x & 0x33333333u) << 2) | ((x >> 2) & 0x33333333u);
    x = ((x & 0x0f0f0f0fu) << 4) | ((x >> 4) & 0x0f0f0f0fu);
    x = ((x & 0x00ff00ffu) << 8) | ((x >> 8) & 0x00ff00ffu);
    x = (x << 16) | (x >> 16);
    return x >> (32 - bits);
}

H2_HD uint32_t ntt_smem_stride(uint32_t logc) { return (1u << logc) + (logc ? 1u : 0u); }
H2_HD uint32_t ntt_smem_bytes(uint32_t sp, uint32_t logc) { return 2u * 16u * (ntt_smem_stride(logc) << sp); }
// + the pass's twiddles (two planes as well): (2^sp - 1) per tile, times the C columns in the last pass
H2_HD uint32_t ntt_twc_bytes(uint32_t sp, uint32_t logc, bool last) { return 32u * ((last ? (1u << logc) : 1u) * ((1u << sp) - 1u)); }

H2_HD fe sm_load(const uint4 *sm, uint32_t plane, uint32_t idx) {
    uint4 lo = sm[idx], hi = sm[plane + idx];
    fe r;
    r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w;
    r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
    return r;
}
H2_HD void sm_store(uint4 *sm, uint32_t plane, uint32_t idx, const fe &a) {
    sm[idx] = make_uint4(a.v[0], a.v[1], a.v[2], a.v[3]);
    sm[plane + idx] = make_uint4(a.v[4], a.v[5], a.v[6], a.v[7]);
}

template <class P> struct NttPass {
    // global natural index j of tile element (r, col)
    static H2_HD uint64_t elem_j(const NttPassArgs &A, uint32_t tile, uint32_t r, uint32_t col) {
        const uint32_t lo = A.log_n - A.s0 - A.sp;
        if (A.flags & NTT_LAST) {     // geometry B (lo == 0)
            uint32_t p_low = (tile << A.logc) | col;
            uint64_t j_high = bitrev32(p_low, A.s0);
            return (j_high << A.sp) | r;
        }
        uint32_t tiles_per_high = 1u << (lo - A.logc);
        uint64_t j_high = tile / tiles_per_high;
        uint64_t jl_block = tile % tiles_per_high;
        return (j_high << (lo + A.sp)) | ((uint64_t)r << lo) | (jl_block << A.logc) | col;
    }
    // low s0 bits of the network position for tile column `col`
    static H2_HD uint32_t p_low_of(const NttPassArgs &A, uint32_t tile, uint32_t col) {
        const uint32_t lo = A.log_n - A.s0 - A.sp;
        if (A.flags & NTT_LAST) return (tile << A.logc) | col;
        uint32_t j_high = tile >> (lo - A.logc);
        return bitrev32(j_high, A.s0);
    }

    static H2_HD void load_phase(const NttPassArgs &A, uint32_t tile, uint32_t tid, uint32_t nthr, uint4 *sm, uint32_t column = 0) {
        const uint32_t R = 1u << A.sp, C = 1u << A.logc, stride = ntt_smem_stride(A.logc), plane = stride << A.sp;
        const fe *in = ntt_col_in(A, column);
        const bool geomB = (A.flags & NTT_LAST) != 0;
        for (uint32_t e = tid; e < R * C; e += nthr) {
            uint32_t r, col;
            if (geomB) { r = e & (R - 1); col = e >> A.sp; } else { col = e & (C - 1); r = e >> A.logc; }
            uint64_t j = elem_j(A, tile, r, col);
            fe x;
            if ((A.flags & NTT_FIRST) && (j >> A.in_log_n) != 0) {
                x = fe_zero();
            } else {
                x = fe_load(in + j);
                if ((A.flags & NTT_FIRST) && (A.flags & NTT_IN_TABLE)) x = fe_mul<P>(x, fe_load(A.in_table + (j & A.in_mask)));
                if ((A.flags & NTT_FIRST) && (A.flags & NTT_IN_SCALE)) x = fe_mul<P>(x, A.in_scale[j % 3]);
            }
            sm_store(sm, plane, r * stride + col, x);
        }
    }

    // one radix-2 stage; sl = 1..sp is the stage number inside this pass
    static H2_HD void stage_phase(const NttPassArgs &A, uint32_t tile, uint32_t sl, uint32_t tid, uint32_t nthr, uint4 *sm) {
        const uint32_t R = 1u << A.sp, C = 1u << A.logc, stride = ntt_smem_stride(A.logc), plane = stride << A.sp;
        const uint32_t d = A.sp - sl;                    // bit of r that this stage pairs on
        const uint32_t tw_shift = A.log_n - A.s0 - sl;   // exponent scale 2^(log_n - s)
        for (uint32_t w = tid; w < (R >> 1) * C; w += nthr) {
            uint32_t col = w & (C - 1), pr = w >> A.logc;
            uint32_t r0 = ((pr >> d) << (d + 1)) | (pr & ((1u << d) - 1u));
            uint32_t r1 = r0 | (1u << d);
            uint32_t k = bitrev32(r0 >> (d + 1), sl - 1);   // p'' mod 2^(sl-1)
            uint64_t e = (((uint64_t)k << A.s0) | p_low_of(A, tile, col)) << tw_shift;
            fe a = sm_load(sm, plane, r0 * stride + col);
            fe b = sm_load(sm, plane, r1 * stride + col);
            fe t = (e == 0) ? b : fe_mul<P>(b, fe_load(A.tw + e));   // tw[0] = 1 (arithmetic.rs:229-236)
            sm_store(sm, plane, r0 * stride + col, fe_add<P>(a, t));
            sm_store(sm, plane, r1 * stride + col, fe_sub<P>(a, t));
        }
    }

    // ---- twiddles of the pass staged in shared memory, stages taken two at a time in registers ---------------------------
    // The twiddle of stage sl (1-based inside the pass) for local index k < 2^(sl-1) is tw[((k << s0) | p_low) << (log_n - s0 - sl)].
    // Geometry A: p_low is a property of the TILE, so a tile needs 2^sp - 1 twiddles, shared by its columns; geometry B: p_low
    // differs per column: C (2^sp - 1).  They are fetched once per tile into `twc` (slot = col_slot (2^sp - 1) + 2^(sl-1) - 1 + k,
    // two 16-byte planes like the data), so the stage loop touches no global memory.
    static H2_HD uint32_t twc_count(const NttPassArgs &A) { return ((A.flags & NTT_LAST) ? (1u << A.logc) : 1u) * ((1u << A.sp) - 1u); }
    static H2_HD uint64_t twc_exponent(const NttPassArgs &A, uint32_t tile, uint32_t slot) {
        const uint32_t per = (1u << A.sp) - 1u;
        const uint32_t cs = slot / per, w = slot % per + 1u;       // w = 2^(sl-1) + k
        uint32_t sl = 1;
        while ((w >> sl) != 0) sl++;
        const uint32_t k = w - (1u << (sl - 1));
        return (((uint64_t)k << A.s0) | p_low_of(A, tile, cs)) << (A.log_n - A.s0 - sl);
    }
    static H2_HD void twiddle_phase(const NttPassArgs &A, uint32_t tile, uint32_t tid, uint32_t nthr, uint4 *twc) {
        const uint32_t total = twc_count(A);
        for (uint32_t slot = tid; slot < total; slot += nthr) sm_store(twc, total, slot, fe_load(A.tw + twc_exponent(A, tile, slot)));
    }
    static H2_HD fe twc_load(const NttPassArgs &A, const uint4 *twc, uint32_t col, uint32_t sl, uint32_t k) {
        const uint32_t per = (1u << A.sp) - 1u;
        return sm_load(twc, twc_count(A), ((A.flags & NTT_LAST) ? col * per : 0u) + (1u << (sl - 1)) - 1u + k);
    }
    static H2_HD uint32_t num_steps(uint32_t sp) { return (sp + 1) / 2; }
    // step `st` = stages 2 st + 1 and 2 st + 2 of the pass (the last step of an odd pass is a single stage).  A radix-4
    // unit holds rows base | {0, 2^(d-1), 2^d, 2^d + 2^(d-1)} of one column in registers: two butterflies of stage sl (pairing
    // bit d = sp - sl, one twiddle), two of stage sl + 1 (pairing bit d - 1, two twiddles) -- half the shared-memory traffic
    // and half the barriers of one stage at a time.  Twiddle 1 (exponent 0, arithmetic.rs:229-236) skips its multiply.
    // L: the shared-memory layout of the tile (element (r, col) -> load / store).
    template <class L>
    static H2_HD void step_phase_l(const NttPassArgs &A, uint32_t tile, uint32_t st, uint32_t tid, uint32_t nthr, const L &lay, const uint4 *twc) {
        const uint32_t R = 1u << A.sp, C = 1u << A.logc;
        const uint32_t sl = 2 * st + 1;
        const bool geomB = (A.flags & NTT_LAST) != 0;
        const bool tile_p0 = !geomB && p_low_of(A, tile, 0) == 0;
        const bool last_step = st + 1 == num_steps(A.sp);
        if (sl == A.sp) {                                   // single last stage: d = 0
            for (uint32_t w = tid; w < (R >> 1) * C; w += nthr) {
                const uint32_t col = w & (C - 1), pr = w >> A.logc;
                const uint32_t r0 = pr << 1, r1 = r0 | 1u;
                const uint32_t k = bitrev32(pr, sl - 1);
                const bool unit = k == 0 && (geomB ? p_low_of(A, tile, col) == 0 : tile_p0);
                fe a = lay.load(A, tile, st, r0, col), b = lay.load(A, tile, st, r1, col);
                fe t = unit ? b : fe_mul<P>(b, twc_load(A, twc, col, sl, k));
                lay.store(A, tile, last_step, r0, col, fe_add<P>(a, t));
                lay.store(A, tile, last_step, r1, col, fe_sub<P>(a, t));
            }
            return;
        }
        const uint32_t d = A.sp - sl;                       // stage sl pairs bit d, stage sl + 1 bit d - 1  (d >= 1)
        for (uint32_t w = tid; w < (R >> 2) * C; w += nthr) {
            const uint32_t col = w & (C - 1), q = w >> A.logc;
            const uint32_t base = ((q >> (d - 1)) << (d + 1)) | (q & ((1u << (d - 1)) - 1u));
            const uint32_t r00 = base, r01 = base | (1u << (d - 1)), r10 = base | (1u << d), r11 = base | (1u << d) | (1u << (d - 1));
            const uint32_t k1 = bitrev32(base >> (d + 1), sl - 1);          // stage sl: both butterflies
            const uint32_t k2a = bitrev32(base >> d, sl);                    // stage sl + 1, rows (00, 01)
            const uint32_t k2b = bitrev32((base >> d) | 1u, sl);             //              rows (10, 11): top bit set, never exponent 0
            const bool p0 = geomB ? p_low_of(A, tile, col) == 0 : tile_p0;
            fe x00 = lay.load(A, tile, st, r00, col), x01 = lay.load(A, tile, st, r01, col);
            fe x10 = lay.load(A, tile, st, r10, col), x11 = lay.load(A, tile, st, r11, col);
            {
                const bool unit = p0 && k1 == 0;
                fe t1 = unit ? fe_zero() : twc_load(A, twc, col, sl, k1);
                fe t = unit ? x10 : fe_mul<P>(x10, t1);
                x10 = fe_sub<P>(x00, t); x00 = fe_add<P>(x00, t);
                t = unit ? x11 : fe_mul<P>(x11, t1);
                x11 = fe_sub<P>(x01, t); x01 = fe_add<P>(x01, t);
            }
            {
                fe t = (p0 && k2a == 0) ? x01 : fe_mul<P>(x01, twc_load(A, twc, col, sl + 1, k2a));
                x01 = fe_sub<P>(x00, t); x00 = fe_add<P>(x00, t);
                t = fe_mul<P>(x11, twc_load(A, twc, col, sl + 1, k2b));
                x11 = fe_sub<P>(x10, t); x10 = fe_add<P>(x10, t);
            }
            lay.store(A, tile, last_step, r00, col, x00); lay.store(A, tile, last_step, r01, col, x01);
            lay.store(A, tile, last_step, r10, col, x10); lay.store(A, tile, last_step, r11, col, x11);
        }
    }
    // the two-plane layout of the classic kernel (row stride C + 1 units)
    struct PlaneLayout {
        uint4 *sm; uint32_t stride, plane;
        H2_HD fe load(const NttPassArgs &, uint32_t, uint32_t, uint32_t r, uint32_t col) const { return sm_load(sm, plane, r * stride + col); }
        H2_HD void store(const NttPassArgs &, uint32_t, bool, uint32_t r, uint32_t col, const fe &x) const { sm_store(sm, plane, r * stride + col, x); }
    };
    static H2_HD void step_phase(const NttPassArgs &A, uint32_t tile, uint32_t st, uint32_t tid, uint32_t nthr, uint4 *sm, const uint4 *twc) {
        PlaneLayout lay;
        lay.sm = sm; lay.stride = ntt_smem_stride(A.logc); lay.plane = lay.stride << A.sp;
        step_phase_l(A, tile, st, tid, nthr, lay, twc);
    }

    static H2_HD void store_phase(const NttPassArgs &A, uint32_t tile, uint32_t tid, uint32_t nthr, const uint4 *sm, uint32_t column = 0) {
        const uint32_t R = 1u << A.sp, C = 1u << A.logc, stride = ntt_smem_stride(A.logc), plane = stride << A.sp;
        fe *out = ntt_col_out(A, column);
        const bool last = (A.flags & NTT_LAST) != 0;
        for (uint32_t e = tid; e < R * C; e += nthr) {
            uint32_t col = e & (C - 1), r = e >> A.logc;
            fe x = sm_load(sm, plane, r * stride + col);
            if (last) {
                uint64_t p = ((uint64_t)bitrev32(r, A.sp) << A.s0) | p_low_of(A, tile, col);
                if (p >= A.out_len) continue;
                if (A.flags & NTT_OUT_SCALE) x = fe_mul<P>(x, A.out_scale[p % 3]);
                if (A.flags & NTT_OUT_PIECES) fe_store(A.out_cols[p >> A.piece_log] + (p & ((1ull << A.piece_log) - 1)), x);
                else fe_store(out + p, x);
            } else {
                fe_store(out + elem_j(A, tile, r, col), x);
            }
        }
    }
};

// Twiddle table: tw[i] = w^i for i < half.  pow2[b] = w^(2^b) (Montgomery), b < 32.
// Thread t produces entries [32 t, 32 t + 32).
template <class P> struct TwiddleGen {
    static H2_HD void pow2_body(fe *pow2, fe omega, uint32_t count) {
        fe w = omega;
        for (uint32_t b = 0; b < count; b++) { fe_store(pow2 + b, w); w = fe_sqr<P>(w); }
    }
    static H2_HD void fill_body(fe *tw, const fe *pow2, uint64_t half, uint64_t t) {
        uint64_t start = t * 32;
        if (start >= half) return;
        fe acc = fe_one<P>();
        uint64_t e = start;
        for (uint32_t b = 5; e >> b; b++)
            if ((e >> b) & 1) acc = fe_mul<P>(acc, fe_load(pow2 + b));
        fe w = fe_load(pow2);
        uint64_t end = start + 32 < half ? start + 32 : half;
        for (uint64_t i = start; i < end; i++) { fe_store(tw + i, acc); acc = fe_mul<P>(acc, w); }
    }
};

#if defined(__CUDACC__)
template <class P> __global__ void __launch_bounds__(128, 4) ntt_pass_kernel(const NttPassArgs A) {
    extern __shared__ uint4 h2_ntt_smem[];
    const uint32_t tile = blockIdx.x, column = blockIdx.y, tid = threadIdx.x, nthr = blockDim.x;
    uint4 *twc = h2_ntt_smem + (ntt_smem_bytes(A.sp, A.logc) >> 4);
    NttPass<P>::twiddle_phase(A, tile, tid, nthr, twc);
    NttPass<P>::load_phase(A, tile, tid, nthr, h2_ntt_smem, column);
    __syncthreads();
    for (uint32_t st = 0; st < NttPass<P>::num_steps(A.sp); st++) {
        NttPass<P>::step_phase(A, tile, st, tid, nthr, h2_ntt_smem, twc);
        __syncthreads();
    }
    NttPass<P>::store_phase(A, tile, tid, nthr, h2_ntt_smem, column);
}
#endif
// ------------------------------------------------------------------------------------------------------------------
// The same pass with the tile traffic on the bulk-copy (TMA) engine: a persistent CTA walks tiles, the rows of tile
// i + 1 land in the second shared-memory buffer (cp.async.bulk global -> shared, completion counted on an mbarrier)
// and the rows of tile i - 1 drain (cp.async.bulk shared -> global) while the warps run the butterflies of tile i, and the
// next tile's twiddles arrive by cp.async.  The compute warps execute no global load or store and no address arithmetic
// per element: one bulk-copy instruction per thread and tile each way.
//   geometry A: a tile row (C adjacent elements, C x 32 B) is contiguous in global memory both ways -> R row copies.
//   geometry B: a tile COLUMN (the 2^sp low indices, 2^sp x 32 B) is contiguous on the way in -> C column copies; the
//       outputs p = bitrev(r) << s0 | p_low are contiguous across the C columns of a row -> the last step writes into a
//       row-major staging area and R row copies carry it out.
// Shared memory is dense (32-byte elements, rows padded by 16 B so that consecutive rows start 4 banks apart).
// ------------------------------------------------------------------------------------------------------------------
H2_HD uint32_t ntt_tma_rowb(uint32_t logc) { return (32u << logc) + 16u; }
H2_HD uint32_t ntt_tma_colb(uint32_t sp) { return (32u << sp) + 16u; }
H2_HD uint32_t ntt_tma_buf_bytes(uint32_t sp, uint32_t logc, bool last) {
    return last ? (ntt_tma_colb(sp) << logc) : (ntt_tma_rowb(logc) << sp);
}
H2_HD uint32_t ntt_tma_smem_bytes(uint32_t sp, uint32_t logc, bool last) {
    return 128u + 2u * ntt_tma_buf_bytes(sp, logc, last) + 2u * ntt_twc_bytes(sp, logc, last) + (last ? (ntt_tma_rowb(logc) << sp) : 0u);
}
H2_HD fe dense_load(const uint8_t *p) {
    const uint4 *q = reinterpret_cast<const uint4 *>(p);
    uint4 lo = q[0], hi = q[1];
    fe r;
    r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w;
    r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
    return r;
}
H2_HD void dense_store(uint8_t *p, const fe &a) {
    uint4 *q = reinterpret_cast<uint4 *>(p);
    q[0] = make_uint4(a.v[0], a.v[1], a.v[2], a.v[3]);
    q[1] = make_uint4(a.v[4], a.v[5], a.v[6], a.v[7]);
}
template <class P> struct NttDense {
    // element (r, col) of the tile in the dense buffers; the first step applies in_scale, the last step out_scale
    struct Layout {
        uint8_t *buf, *out;          // out: geometry B's row-major staging (last step), else == buf
        uint32_t rowb, colb;
        bool geomB;
        H2_HD fe load(const NttPassArgs &A, uint32_t tile, uint32_t st, uint32_t r, uint32_t col) const {
            fe x = dense_load(geomB ? buf + col * colb + r * 32u : buf + r * rowb + col * 32u);
            if (st == 0 && (A.flags & NTT_FIRST) && (A.flags & NTT_IN_SCALE)) x = fe_mul<P>(x, A.in_scale[NttPass<P>::elem_j(A, tile, r, col) % 3]);
            return x;
        }
        H2_HD void store(const NttPassArgs &A, uint32_t tile, bool last_step, uint32_t r, uint32_t col, const fe &x) const {
            if (last_step && geomB) {
                fe y = x;
                if (A.flags & NTT_OUT_SCALE) {
                    const uint64_t p = ((uint64_t)bitrev32(r, A.sp) << A.s0) | NttPass<P>::p_low_of(A, tile, col);
                    y = fe_mul<P>(y, A.out_scale[p % 3]);
                }
                dense_store(out + r * rowb + col * 32u, y);
            } else dense_store(geomB ? buf + col * colb + r * 32u : buf + r * rowb + col * 32u, x);
        }
    };
    // what the copy engine moves for one tile.  Copy unit u: geometry A -> row u (u < R); geometry B in -> column u (u < C),
    // geometry B out -> row u (u < R).  `valid` = false: nothing to copy (zero padding in, truncated out).
    struct Span { uint64_t elem; uint32_t smem_off, bytes; bool valid; };
    static H2_HD uint32_t in_units(const NttPassArgs &A) { return (A.flags & NTT_LAST) ? (1u << A.logc) : (1u << A.sp); }
    static H2_HD Span in_span(const NttPassArgs &A, uint32_t tile, uint32_t u) {
        Span s;
        const bool geomB = (A.flags & NTT_LAST) != 0;
        s.elem = geomB ? NttPass<P>::elem_j(A, tile, 0, u) : NttPass<P>::elem_j(A, tile, u, 0);
        s.smem_off = geomB ? u * ntt_tma_colb(A.sp) : u * ntt_tma_rowb(A.logc);
        s.bytes = geomB ? (32u << A.sp) : (32u << A.logc);
        s.valid = !((A.flags & NTT_FIRST) && (s.elem >> A.in_log_n) != 0);     // runs never straddle 2^in_log_n (powers of two)
        return s;
    }
    static H2_HD Span out_span(const NttPassArgs &A, uint32_t tile, uint32_t r) {
        Span s;
        s.smem_off = r * ntt_tma_rowb(A.logc);
        s.bytes = 32u << A.logc;
        if (A.flags & NTT_LAST) {
            s.elem = ((uint64_t)bitrev32(r, A.sp) << A.s0) | NttPass<P>::p_low_of(A, tile, 0);
            s.valid = s.elem < A.out_len;
        } else { s.elem = NttPass<P>::elem_j(A, tile, r, 0); s.valid = true; }
        return s;
    }
    static H2_HD bool supported(const NttPassArgs &A) {
        if ((A.flags & NTT_LAST) && (A.out_len & ((1ull << A.logc) - 1))) return false;      // whole rows only on the way out
        if ((A.flags & NTT_FIRST) && (A.flags & NTT_LAST)) return false;                      // single-pass transforms: classic kernel
        if (A.flags & (NTT_IN_TABLE | NTT_OUT_PIECES)) return false;                          // the vanishing quotient's fusions: classic kernel
        return true;
    }
};

#if defined(__CUDACC__)
namespace tma {
__device__ __forceinline__ uint32_t saddr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(saddr(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(saddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(saddr(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(saddr(dst)), "l"(src), "r"(bytes),
                 "r"(saddr(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void *dst, const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(saddr(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void cp16(void *dst, const void *src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(saddr(dst)), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
}  // namespace tma

template <class P> __global__ void __launch_bounds__(128, 4) ntt_pass_tma_kernel(const NttPassArgs A, uint32_t tiles) {
    extern __shared__ __align__(128) uint8_t h2_ntt_tma_smem[];
    const uint32_t tid = threadIdx.x, nthr = blockDim.x;
    const bool geomB = (A.flags & NTT_LAST) != 0;
    const uint32_t R = 1u << A.sp, bufb = ntt_tma_buf_bytes(A.sp, A.logc, geomB), twb = ntt_twc_bytes(A.sp, A.logc, geomB);
    uint64_t *full = reinterpret_cast<uint64_t *>(h2_ntt_tma_smem);                 // full[0], full[1]
    uint8_t *buf0 = h2_ntt_tma_smem + 128;
    uint8_t *twc0 = buf0 + 2 * bufb;
    uint8_t *outst = twc0 + 2 * twb;                                                 // geometry B only
    const uint32_t ntw = NttPass<P>::twc_count(A);
    const uint32_t units_in = NttDense<P>::in_units(A);
    const fe *in = ntt_col_in(A, blockIdx.y);           // grid.y: the column, as in ntt_pass_kernel
    fe *out = ntt_col_out(A, blockIdx.y);
    if (tid == 0) {   // one arrival per copy unit: every issuing thread announces its own bytes
        tma::mbar_init(&full[0], units_in);
        tma::mbar_init(&full[1], units_in);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // everything one tile needs, issued asynchronously: rows / columns by the bulk-copy engine, twiddles by cp.async
    auto fetch = [&](uint32_t tile, uint32_t b) {
        uint8_t *buf = buf0 + b * bufb;
        for (uint32_t u = tid; u < units_in; u += nthr) {
            const auto sp_ = NttDense<P>::in_span(A, tile, u);
            if (sp_.valid) {
                tma::mbar_expect_tx(&full[b], sp_.bytes);
                tma::bulk_g2s(buf + sp_.smem_off, in + sp_.elem, sp_.bytes, &full[b]);
            } else {
                for (uint32_t o = 0; o < sp_.bytes; o += 16) *reinterpret_cast<uint4 *>(buf + sp_.smem_off + o) = make_uint4(0, 0, 0, 0);
                tma::mbar_expect_tx(&full[b], 0);          // zero padding: arrive without bytes (the release orders the stores above)
            }
        }
        uint4 *twc = reinterpret_cast<uint4 *>(twc0 + b * twb);
        for (uint32_t slot = tid; slot < ntw; slot += nthr) {
            const fe *src = A.tw + NttPass<P>::twc_exponent(A, tile, slot);
            tma::cp16(twc + slot, src);
            tma::cp16(twc + ntw + slot, reinterpret_cast<const uint8_t *>(src) + 16);
        }
        tma::cp_commit();
    };
    uint32_t cur = blockIdx.x;
    if (cur < tiles) fetch(cur, 0);
    for (uint32_t it = 0; cur < tiles; it++, cur += gridDim.x) {
        const uint32_t b = it & 1u, nxt = cur + gridDim.x;
        // this thread's stores of the previous tile have finished READING shared memory: its rows of the other buffer (geometry
        // A) / of the staging area (geometry B) may be overwritten
        tma::bulk_wait_read0();
        if (nxt < tiles) { fetch(nxt, b ^ 1u); tma::cp_wait<1>(); } else tma::cp_wait<0>();
        tma::mbar_wait(&full[b], (it >> 1) & 1u);
        __syncthreads();
        typename NttDense<P>::Layout lay;
        lay.buf = buf0 + b * bufb; lay.out = geomB ? outst : lay.buf;
        lay.rowb = ntt_tma_rowb(A.logc); lay.colb = ntt_tma_colb(A.sp); lay.geomB = geomB;
        const uint4 *twc = reinterpret_cast<const uint4 *>(twc0 + b * twb);
        for (uint32_t st = 0; st < NttPass<P>::num_steps(A.sp); st++) {
            NttPass<P>::step_phase_l(A, cur, st, tid, nthr, lay, twc);
            if (st + 1 < NttPass<P>::num_steps(A.sp)) __syncthreads();
        }
        tma::fence_async_smem();          // the generic-proxy writes above become visible to the bulk-copy engine
        __syncthreads();
        for (uint32_t r = tid; r < R; r += nthr) {
            const auto sp_ = NttDense<P>::out_span(A, cur, r);
            if (sp_.valid) tma::bulk_s2g(out + sp_.elem, lay.out + sp_.smem_off, sp_.bytes);
        }
        tma::bulk_commit();
    }
    tma::bulk_wait0();
}
#endif

#if defined(__CUDACC__)
template <class P> __global__ void twiddle_pow2_kernel(fe *pow2, fe omega, uint32_t count) {
    if (threadIdx.x == 0 && blockIdx.x == 0) TwiddleGen<P>::pow2_body(pow2, omega, count);
}
template <class P> __global__ void twiddle_fill_kernel(fe *tw, const fe *pow2, uint64_t half) {
    TwiddleGen<P>::fill_body(tw, pow2, half, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
// elementwise conversions used at the ABI boundary
template <class P> __global__ void fe_scale_kernel(fe *a, uint64_t n, fe c) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fe_store(a + i, fe_mul<P>(fe_load(a + i), c));
}
#endif

// Host-side pass planning (shared with the emulation).  Returns the number of passes and fills
// sp[] / logc[]; tiles hold at most 2^H2_NTT_TILE_LOG elements.
// 512-element tiles, 128 threads: ~7 CTAs/SM, 2^20 -> 2048 tiles = 2.2 waves of 132 x 7.  1024-element tiles (1.1 waves) are
// slower on an H100 (400 W limit) despite the fuller last wave: 2^16 0.038 vs 0.031 ms, 2^20 0.273 vs 0.256 ms, equal at 2^22 / 2^24
#define H2_NTT_TILE_LOG 9
#define H2_NTT_MAX_SP 7
inline int ntt_plan(uint32_t log_n, uint32_t sp[8], uint32_t logc[8]) {
    if (log_n == 0) return 0;
    if (log_n <= H2_NTT_TILE_LOG + 1) { sp[0] = log_n; logc[0] = 0; return 1; }   // single CTA, up to 1024 elements
    int passes = (int)((log_n + H2_NTT_MAX_SP - 1) / H2_NTT_MAX_SP);
    uint32_t base = log_n / passes, rem = log_n % passes, s0 = 0;
    for (int i = 0; i < passes; i++) {
        sp[i] = base + ((uint32_t)i < rem ? 1u : 0u);
        uint32_t lo = log_n - s0 - sp[i];
        uint32_t lc = H2_NTT_TILE_LOG - sp[i];
        if (lc > 4) lc = 4;
        if (i == passes - 1) { if (lc > s0) lc = s0; } else { if (lc > lo) lc = lo; }
        logc[i] = lc;
        s0 += sp[i];
    }
    return passes;
}
// Column batches: each pass of a transform of `count` columns of one size and domain is one launch whose grid.y is the
// column.  A multi-pass transform keeps its intermediate data in scratch, one 2^log_n-element slot per column: a group
// takes as many columns as fit in H2_NTT_BATCH_SCRATCH bytes (at least one, at most 65535, the grid.y limit), so the scratch
// is at most max(32 * 2^log_n, H2_NTT_BATCH_SCRATCH) bytes for any count.  Single-pass transforms need no scratch.
#define H2_NTT_BATCH_SCRATCH (1ull << 28)
inline uint64_t ntt_group(uint32_t log_n, int passes, uint64_t count) {
    uint64_t g = passes > 1 ? H2_NTT_BATCH_SCRATCH / (32ull << log_n) : count;
    if (g < 1) g = 1;
    if (g > 65535) g = 65535;
    return g < count ? g : count;
}
// The size arguments of h2_poly_vanishing_quotient (K24): `count` pieces of 2^k coefficients out of an extended domain of
// 2^ext_k points, t_len inverses of t(X) = X^n - 1 repeated over it.  The reason they are rejected, or nullptr.
inline const char *vanishing_quotient_sizes(uint32_t k, uint32_t ext_k, uint64_t count, uint32_t t_len) {
    if (ext_k > 30) return "ext_k > 30";
    if (ext_k < k) return "ext_k < k";
    if (count == 0 || count > (1ull << (ext_k - k))) return "count must be at least 1 and count * 2^k at most 2^ext_k";
    if (t_len == 0 || (t_len & (t_len - 1)) || t_len > (1u << ext_k)) return "t_len must be a power of two <= 2^ext_k";
    return nullptr;
}

}  // namespace h2
