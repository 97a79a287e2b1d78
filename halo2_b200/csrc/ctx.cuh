// Host-side context shared by the translation units of the C ABI (capi_*.cu): error reporting, device buffers, the per-device
// Context, launch / profiling helpers.  The library is split into several TUs so that they compile in parallel and a change
// to one kernel family rebuilds one of them; every kernel is a template (or inline) in a header, so each TU instantiates
// what it launches.  No torch types.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/halo2_b200.h"
#define H2_MAX_UPLOAD_CHUNKS 4
#define H2_MAX_DEVICES 16
#include "curve.cuh"

using namespace h2;

// ------------------------------------------------------------------------------------------------
// errors, context
// ------------------------------------------------------------------------------------------------
int fail(const std::string &m);          // sets the calling thread's last error, returns 1
const std::string &last_error_string();  // the calling thread's last error (worker threads hand theirs to the caller)
#define CU(expr)                                                                                         \
    do {                                                                                                 \
        cudaError_t e_ = (expr);                                                                         \
        if (e_ != cudaSuccess) return fail(std::string(#expr) + ": " + cudaGetErrorString(e_));          \
    } while (0)

// Cached CUDA graphs (fixed-base MSMs) hold raw pointers into the library's scratch pools and window tables: every
// (re)allocation or release of a TRACKED buffer bumps the generation and invalidates them.  Buffers a graph can only see
// through its key (caller polynomials, IPA session vectors: the scalars / out pointers are part of the key) are untracked --
// allocating a ResidentPoly between two commits must not throw the commit graphs away.
extern std::atomic<uint64_t> g_alloc_gen;
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    bool tracked = true;
    int ensure(size_t bytes) {
        if (bytes <= cap) return 0;
        if (tracked) g_alloc_gen++;
        if (p) { cudaFree(p); p = nullptr; cap = 0; }
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { p = nullptr; return fail(std::string("cudaMalloc(") + std::to_string(want) + "): " + cudaGetErrorString(e)); }
        cap = want;
        return 0;
    }
    void release() { if (p) { cudaFree(p); if (tracked) g_alloc_gen++; } p = nullptr; cap = 0; }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};


struct TwiddleEntry { int field; uint32_t log_n; uint8_t omega[32]; DevBuf buf; uint64_t stamp; };
struct BaseSet {
    int curve; size_t n; DevBuf buf;
    DevBuf table; uint32_t c = 0, W = 0;   // W x n window shifts 2^(c w) G_i (bucket method over one shared bucket set)
    DevBuf dtable;                         // 32 x 128 x n digit multiples m 2^(8 w) G_i (fixedbase.cuh: direct sum, small sets)
    uint32_t users = 0;                    // registered sets (g_bases): calls in flight on any lane that read the set (BasesRef)
    uint32_t sessions = 0;                 // ... and open IPA sessions on any lane that refer to it; both under g_reg_mu
};

struct PolyBuf {                           // device-resident polynomial, Montgomery form, len + 1 slots
    int field; size_t len; DevBuf buf;
    uint32_t users = 0;                    // shared polynomials (g_shared_polys): calls in flight on any context that read it (PolyArgs); under g_reg_mu
    PolyBuf() { buf.tracked = false; }
};
struct IpaSession {
    uint64_t bases; uint32_t k, round; int folded; DevBuf p, b, s, scal, out;
    IpaSession() { p.tracked = b.tracked = s.tracked = scal.tracked = out.tracked = false; }
};

// A fixed-base MSM over resident bases is ~25 small launches whose parameters repeat call after call (same table, same
// scratch, same sizes): the second call with a given key is captured into a CUDA graph, later ones replay it.
struct MsmGraph {
    const void *scalars, *bases, *out;
    size_t n; uint64_t stride, gen;
    uint32_t c, sets; int scalars_mont, out_canonical;
    uint32_t fast = 0;
    uint32_t seen = 0; uint64_t launches = 0, stamp = 0;
    cudaGraphExec_t exec = nullptr;
};

// Pinned staging ring for transfers from / to PAGEABLE caller memory (a Rust Vec, a numpy array): a plain cudaMemcpyAsync
// from pageable memory is staged by the driver through one thread and runs at a fraction of the link rate, and it blocks
// the caller so nothing overlaps.  Here a small pool of host threads copies slot-sized pieces into pinned slots while the
// DMA engine drains the previous ones (capi_core.cu: upload_async / download_sync).
struct StageRing {
    enum { SLOTS = 4 };
    uint8_t *slot[SLOTS] = {};
    size_t slot_bytes = 0;
    cudaEvent_t done[SLOTS] = {};
    bool busy[SLOTS] = {};
    uint32_t next = 0;
    int ensure();
    void destroy();
};

// The mutex of a Context.  Copying or assigning a Context (ctx_destroy resets one with `C = Context()`) leaves it alone.
struct CtxMutex {
    std::mutex m;
    CtxMutex() {}
    CtxMutex(const CtxMutex &) {}
    CtxMutex &operator=(const CtxMutex &) { return *this; }
};

struct Context {
    CtxMutex mu;                             // held for a whole call on this context (CtxLock)
    bool ready = false;
    int device = -1;
    // Every call's work, in call order.  The context's device state (scratch, caches, tables, graphs, resident polynomials, IPA
    // sessions) is touched only on this stream, on copy_stream under its events (msm_host_common), by a multi-GPU worker's peer
    // copy into the primary's multi_parts (synchronised in msm_pass before the worker returns), or on a caller's stream inside a
    // StreamSplice.  A new entry point that takes a caller's stream and touches context state must use the splice.
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;      // uploads that may overlap compute (bases of a one-shot MSM)
    cudaEvent_t ev_scalars_up = nullptr, ev_bases_up[H2_MAX_UPLOAD_CHUNKS] = {}, ev_scal_up[H2_MAX_UPLOAD_CHUNKS] = {};
    uint32_t chunk_min_log = 19;             // one-shot MSMs of >= 2^19 points upload their bases in chunks
    cudaEvent_t ev_splice = nullptr;         // StreamSplice
    uint32_t window_override = 0;
    const uint32_t *last_flags = nullptr;    // device flags of the most recent MSM (test hook; the fast fixed-base pass's validity check)
    uint32_t fast_on = 1;                    // fixed-base passes over resident tables first run WITHOUT the fallback kernels (exact sort: histogram, 3 scan
                                             // kernels, scatter; partial merges: 3 kernels) and their two memsets -- 10 of ~27 graph nodes that do nothing on
                                             // ordinary inputs; the two device flags come back with the result and a set flag re-runs the full pass
    uint64_t natural_max_buckets = 1ull << 14;   // fast passes with up to this many buckets take them in index order (MsmPlan::natural).  At k = 14
                                             // (one lane pair per bucket) 2^14 buckets are a single commit, 2^15 an IPA round's two sets and 2^16 four
                                             // batched commits: only a pass that is resident at once gains
    uint32_t last_plan[8] = {};              // what the most recent MSM pass ran, recorded on the host (h2_test_last_msm_plan)
    bool have_plan = false;
    uint32_t *h_flags = nullptr;             // pinned host copy of the two flags
    uint32_t sort_bins = 1;                  // single-pass binned sort (0: always the exact two-pass sort)
    uint32_t glv_on = 1;                     // GLV endomorphism split for one-shot / table-less MSMs
    uint32_t accum_ways = 12;                // lanes per work item in the small-problem accumulation: 12 (default) / 14 = 2 / 4 INDEPENDENT lanes, each adding every
                                             // 2nd / 4th reference serially, partial sums folded by shuffles (msm_accum0_split_kernel); 0 = a cooperating PAIR
                                             // (10 lane-multiplies per addition, 5 levels); 1 / 2 / 4 = quads.  A cooperative addition is no shorter than a serial
                                             // one in practice, so cutting the longest bucket's chain in two is what helps
    uint32_t poly_cta = 0;                   // 1: eval_polynomial / kate_division of polynomials up to 2^16 coefficients in one CTA each; 0 (default): the level
                                             // tree -- one CTA's 16-64-step serial slices lose to three launches that fill the machine
    uint64_t small_accum_refs = 1ull << 20;  // MSMs with up to this many references accumulate with cooperating lanes (accum_ways); larger ones with a thread per item
    uint32_t ntt_tma = 0;                    // NTT passes: 1 = bulk-copy (TMA) persistent kernel where it applies, 0 = classic kernel.  Measured on
                                             // an H100 SXM (700 W, tools/ntt_time.py): 2^20 0.310 vs 0.254 ms, 2^24 5.36 vs 4.21 ms -- the pass is bound by the
                                             // integer pipes, not by its memory phases (pipe utilisation not profiled on H100), and
                                             // the double-buffered tiles cost occupancy (4 CTAs/SM, 2 in the last pass): opt-in, default off
    uint32_t ba_variant = 3;                 // kernel variant of the rounds (tuning): 0 / 1 = gather chunks of 4 pairs at 4 / 5 CTAs per SM, 2 / 3 = chunks of 2
    uint32_t ba_rounds = 0, ba_target = 32;  // batched-affine halving rounds ahead of the XYZZ accumulation of large one-shot MSMs and the pairs per thread
                                             // one inversion is shared by (h2_test_set_batched_affine).  OFF by default -- measured on an H100 SXM (700 W,
                                             // tools/ba_sweep.py): best setting (variant 2, 1 round, 32 pairs) 4.88 ms vs 4.31 ms without at 2^20, 18.9 vs
                                             // 16.2 ms at 2^22; 2 / 3 rounds slower still.  An affine addition is 6 multiplies instead of 10 but not fewer instructions
                                             // (field add/sub, the inversion's share, call marshalling, local-memory products), and its dependent
                                             // reference -> point gathers leave the kernel latency-bound at 14-20 warps per SM (DESIGN.md K4a)
    uint32_t ecfft_quad = 1;                 // EC-FFT butterfly form: 1 = by size (default), 0 = one thread each, 2 = quads (test hook)
    // MSM scratch
    DevBuf scal_in, bases_in, bases_phi, glv_parts, scal_canon, counts, cursor, refs, size_hist, items, bucket_sum, pkey, pstart, pend, ppt, ra_t, ra_e, r0, r1,
        wsum, scan_blocks, result, misc, ba_lv[3];
    // NTT scratch
    DevBuf ntt_io, ntt_out, ntt_work, pow2;
    DevBuf col_tab;                          // the column table of the call in flight (col_table)
    // EC-FFT / batch-normalise scratch: XYZZ work array (128 B per point), staging for the host forms
    DevBuf ec_work, ec_io, ec_out;
    DevBuf fb_a, fb_b;                       // partial sums of the direct-sum fixed-base MSM (ping-pong)
    DevBuf multi_parts;                      // primary device: the per-GPU partial results of a multi-GPU MSM (peer-written)
    StageRing stage;
    DevBuf ast_code, ast_consts;             // asteval.cuh: the postfix program and its constants
    DevBuf po_lvl, po_q, po_pts;             // polyops.cuh: level arrays, kate carries, per-level points
    DevBuf lk_keys, lk_u32;                  // lookup.cuh: sorted tables, histogram / scan / leftover arrays
    DevBuf kg_tab, kg_map;                   // keygen.cuh: power tables + error word, one piece of the copy-constraint mapping (all of it for assembly.cuh)
    DevBuf as_edge, as_cell, as_slot;        // assembly.cuh: per-copy, per-cell and per-slot u32 arrays
    DevBuf gp_val, gp_aux;                   // grandproduct.cuh: denominators / mv of every column, power tables + carries
    std::vector<TwiddleEntry *> twiddles;
    uint64_t tw_stamp = 0;
    std::map<uint64_t, BaseSet *> shards;    // this device's shards of multi-GPU base sets (h2_multi_bases_register)
    std::map<uint64_t, IpaSession *> ipa;
    std::map<uint64_t, PolyBuf *> polys;
    std::vector<MsmGraph> graphs;
    uint64_t graph_stamp = 0;
    uint32_t graphs_on = 1;
    std::vector<PolyBuf *> poly_pool;        // freed resident polynomials keep their buffers for the next h2_poly_alloc of that size
    size_t poly_pool_bytes = 0;
    std::vector<IpaSession *> ipa_pool;      // finished sessions keep their buffers for the next proof (no cudaMalloc per opening)
};
// One Context per CUDA device, plus up to H2_MAX_LANES lanes: extra contexts on the primary device, each with its own
// streams, scratch, caches, settings, resident polynomials and IPA sessions, so that independent provers on different host
// threads run concurrently (h2_lane_create / h2_lane_bind).  API functions work on the context the calling thread's
// g_cur points at: its bound lane, or the PRIMARY context (the device h2_init bound) when it never bound one.  The multi-GPU
// entry points (h2_multi_*) run one worker thread per device, each of which points its g_cur at its device's context
// while the calling thread holds the primary's mutex -- so all the single-GPU code below runs unchanged, concurrently, on
// every device and every lane.
//
// Locks, outermost first; a thread never takes one while holding a later one:
//   1. g_life_mu      h2_init, h2_shutdown, h2_multi_init, h2_lane_create, h2_lane_destroy
//   2. Context::mu    a call on that context, for the whole call.  A thread holds one at a time, except h2_shutdown, which
//                     takes the primary's and then every live lane's in slot order (every other holder finishes its call
//                     without waiting for a second context)
//   3. g_reg_mu       the lane table and bindings, the shared base sets (g_bases), the shared polynomials (g_shared_polys) and
//                     their user counts, g_multi, g_multi_bases; held for map lookups only, never while taking a Context
//                     mutex.  h2_bases_release and h2_poly_free of a shared polynomial hold no Context mutex: they wait on
//                     g_users_cv under it for the object's users, which drop them without taking a second context
// Handles of base sets, polynomials, IPA sessions, multi-GPU base sets and lanes come from one process-wide counter
// (new_handle) that h2_shutdown does not reset: a handle names one object of one kind on one lane, and any other use of it
// -- a foreign lane, a stale handle from before a shutdown -- finds nothing and is reported as unknown.  A shared
// polynomial (h2_poly_share) keeps its handle and is then known, for reading only, on every lane.
#define H2_MAX_LANES 16
extern Context g_ctxs[H2_MAX_DEVICES];
extern Context g_lanes[H2_MAX_LANES];
extern Context *g_primary;
extern thread_local Context *g_cur;
extern thread_local uint64_t g_cur_epoch;    // g_epoch when g_cur was set
extern std::atomic<uint64_t> g_epoch;        // bumped by h2_shutdown: a lane bound before it is gone
extern Context g_dead;                       // never ready: what a thread whose lane h2_shutdown destroyed works on
static inline Context &cur_ctx() {
    if (!g_cur) return *g_primary;
    if (g_cur_epoch != g_epoch.load(std::memory_order_relaxed)) return g_dead;
    return *g_cur;
}
static inline void set_cur(Context *c) { g_cur = c; g_cur_epoch = g_epoch.load(); }
#define g_ctx (cur_ctx())
extern std::mutex g_life_mu, g_reg_mu;
struct CtxLock {                             // the calling thread's context, for the whole call
    std::lock_guard<std::mutex> g;
    CtxLock() : g(cur_ctx().mu.m) {}
};
uint64_t new_handle();
bool on_lane();                              // the calling thread is bound to a lane (not the primary context)
// Shared base sets (h2_bases_register*): registered once, read by every lane.  A BasesRef holds the set for one call; the
// set cannot be released before it is dropped.
extern std::map<uint64_t, BaseSet *> g_bases;
struct BasesRef {
    BaseSet *b = nullptr;
    explicit BasesRef(uint64_t handle, bool open_session = false);   // b == nullptr: unknown handle
    ~BasesRef();
    BasesRef(const BasesRef &) = delete;
    BasesRef &operator=(const BasesRef &) = delete;
};
void bases_session_end(uint64_t handle);     // an IPA session on the set finished (or its lane was destroyed)
// optional per-kernel timing (bench.py's roofline leg): event pairs recorded on the launch stream
struct ProfSpan { int kind; cudaEvent_t e0, e1; };
extern std::atomic<bool> g_prof_on;
extern std::vector<ProfSpan> g_prof;
enum { PROF_MSM_ACCUM0 = 0, PROF_NTT_PASS = 1, PROF_KINDS = 2 };
void prof_begin(int kind, cudaStream_t s);
void prof_end(cudaStream_t s);
extern std::atomic<uint64_t> g_launches;

#define LAUNCH(kernel, grid, block, smem, stream, ...)                                                   \
    do {                                                                                                 \
        kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                                      \
        g_launches.fetch_add(1, std::memory_order_relaxed);                                              \
        cudaError_t e_ = cudaGetLastError();                                                             \
        if (e_ != cudaSuccess) return fail(std::string(#kernel) + " launch: " + cudaGetErrorString(e_)); \
    } while (0)

// Host -> device copy on stream `s` that keeps the link busy whatever the caller's memory is: pinned / registered memory
// goes straight to cudaMemcpyAsync (the source must then stay valid until the stream has run it -- every caller synchronises
// before returning); pageable memory goes through the context's pinned ring and has been fully READ when this returns.
int upload_async(void *d_dst, const void *h_src, size_t bytes, cudaStream_t s);
// Device -> host copy ordered behind the work already on `s`; returns when the data is in h_dst.
int download_sync(void *h_dst, const void *d_src, size_t bytes, cudaStream_t s);
void h2_set_staging(int on);             // test / bench hook: 0 = always plain cudaMemcpyAsync
int require_ready();
// One call on a caller's stream `s` that uses the calling context's state (scratch, the twiddle cache, pow2) while its kernels
// stay on `s`: on construction `s` waits for the work queued so far on the context's stream, and on destruction, whichever
// way the call returns, the context's stream waits for what the call queued on `s`.  One event serves both waits, as a wait
// takes the event's state when it is issued and the context's mutex keeps other calls from recording it in between.
// `failed`: the entry wait could not be issued (the error is set), and the call returns without using `s`.
struct StreamSplice {
    explicit StreamSplice(cudaStream_t s);
    ~StreamSplice();
    StreamSplice(const StreamSplice &) = delete;
    StreamSplice &operator=(const StreamSplice &) = delete;
    Context &X;
    cudaStream_t s;
    int failed = 0;
};
static inline uint32_t blocks_for(uint64_t n, uint32_t bs) { return (uint32_t)((n + bs - 1) / bs); }

// The host-side field elements and points of one entry point `who`, in the encoding `repr` (include/halo2_b200.h).
// check() runs before the call copies or launches anything:
//   - repr is H2_REPR_CANONICAL or H2_REPR_MONTGOMERY, else "<who>: unknown repr";
//   - every required host pointer is set, else "<who>: null <name>" (name as in the header); a Need whose `required` is
//     false (an optional pointer, or an array of no elements) is not checked.
// Then a single element is read into Montgomery form (elem), an array goes to the device and into Montgomery form (up, or
// to_mont after a copy of the caller's own), and device elements come back in repr (down from resident data, which stays
// in Montgomery form; from_mont on scratch).  canon() / mont() are for kernels that take the encoding as a flag.
struct HostArgs {
    struct Need { const void *p; const char *name; bool required = true; };
    HostArgs(const char *who, int repr) : who(who), repr(repr) {}
    int check(std::initializer_list<Need> needs = {}) const;
    bool canon() const { return repr == H2_REPR_CANONICAL; }
    bool mont() const { return repr == H2_REPR_MONTGOMERY; }
    template <class P> fe elem(const void *bytes) const {
        fe x;
        memcpy(x.v, bytes, 32);
        return mont() ? x : fe_to_mont<P>(x);
    }
    int up(int field, fe *d, const void *h, size_t n, cudaStream_t s) const;   // upload_async, then to_mont
    int to_mont(int field, fe *d, size_t n, cudaStream_t s) const;             // device elements in repr -> Montgomery, in place
    int from_mont(int field, fe *d, size_t n, cudaStream_t s) const;           // Montgomery -> repr, in place (scratch only)
    int down(int field, void *h, const fe *d, size_t n, cudaStream_t s) const; // to the host in repr; canonical converts a scratch copy
    const char *who;
    int repr;
};
// Shared polynomials (h2_poly_share): read-only from then on, and readable from every context.  Sharing moves them out of
// their owner's `polys` into this registry with unchanged handles; they never go into a poly_pool.
extern std::map<uint64_t, PolyBuf *> g_shared_polys;
// The resident-polynomial arguments of one entry point `who`, all checked before it launches anything.  `name` is the
// parameter's name as the header spells it; an element of a handle array is "<name>[i]".
//   - an output is a polynomial of the calling context; a shared one fails with "the polynomial is shared (read-only)";
//   - an input is the calling context's or a shared one, and a shared input counts the call as a user until the PolyArgs is
//     dropped, so h2_poly_free cannot free it meanwhile.  Declared after the call's CtxLock, so it is dropped before the
//     context's mutex;
//   - every polynomial is over one field (`field`, the curve's scalar field for the MSM-side calls, or else the first
//     polynomial's) and holds the elements [off, off + len) its lookup asks for (off = 0 unless given), else "a polynomial
//     holds fewer than <len_name> elements".  off + len is never formed, so it cannot wrap;
//   - with distinct(), no output is listed twice or is also an input: "<a> is also <b>", the output first ("dst[2] is also
//     dst[0]", "dst is also src").  A call that works in place names its index-paired output and input arrays, and then
//     out[i] == in[i] is allowed.
// A failed lookup sets "<who>: <reason>" for a single handle, "<who>: <name>[i]: <reason>" for an element of an array; a
// lookup then gives nullptr, the other members 1.
struct PolyArgs {
    explicit PolyArgs(const char *who, int field = -1) : who(who), field(field), field_given(field >= 0) {}
    ~PolyArgs();
    PolyBuf *out(uint64_t h, const char *name, uint64_t off, uint64_t len, const char *len_name) { return find(true, h, name, -1, off, len, len_name); }
    PolyBuf *in(uint64_t h, const char *name, uint64_t off, uint64_t len, const char *len_name) { return find(false, h, name, -1, off, len, len_name); }
    PolyBuf *out(uint64_t h, const char *name, uint64_t len, const char *len_name) { return out(h, name, 0, len, len_name); }
    PolyBuf *in(uint64_t h, const char *name, uint64_t len, const char *len_name) { return in(h, name, 0, len, len_name); }
    using Polys = std::vector<PolyBuf *>;    // handle arrays: h[0 .. n) into v
    int out(const uint64_t *h, size_t n, const char *name, uint64_t off, uint64_t len, const char *len_name, Polys &v) { return find(true, h, n, name, off, len, len_name, v); }
    int out(const uint64_t *h, size_t n, const char *name, uint64_t len, const char *len_name, Polys &v) { return find(true, h, n, name, 0, len, len_name, v); }
    int in(const uint64_t *h, size_t n, const char *name, uint64_t len, const char *len_name, Polys &v) { return find(false, h, n, name, 0, len, len_name, v); }
    // element i holds at least lens[i] elements ("a polynomial holds fewer than <len_name>[i] elements")
    int out(const uint64_t *h, size_t n, const char *name, const size_t *lens, const char *len_name, Polys &v) { return find(true, h, n, name, lens, len_name, v); }
    int in(const uint64_t *h, size_t n, const char *name, const size_t *lens, const char *len_name, Polys &v) { return find(false, h, n, name, lens, len_name, v); }
    int distinct(const char *in_place_out = nullptr, const char *in_place_in = nullptr);
    PolyArgs(const PolyArgs &) = delete;
    PolyArgs &operator=(const PolyArgs &) = delete;

  private:
    struct Arg { PolyBuf *p; bool out; const char *name; int64_t i; };   // i < 0: a single handle
    std::string who;
    int field;
    bool field_given;
    std::vector<Arg> args;                   // every polynomial looked up, in order
    std::vector<PolyBuf *> held;             // the shared polynomials this call is a user of
    PolyBuf *find(bool out, uint64_t h, const char *name, int64_t i, uint64_t off, uint64_t len, const char *len_name);
    int find(bool out, const uint64_t *h, size_t n, const char *name, uint64_t off, uint64_t len, const char *len_name, Polys &v);
    int find(bool out, const uint64_t *h, size_t n, const char *name, const size_t *lens, const char *len_name, Polys &v);
};
// One upload of a kernel's column table into the context's table buffer (col_tab), on `s`: the device
// pointers of `cols` in the order the kernel reads them (a null PolyBuf gives a null pointer), then `bytes` host bytes from
// `data` at the next 32-byte boundary.  The table is scratch: it holds for the kernels the call queues on `s` after it.
struct ColTable {
    fe *const *cols;                         // the pointers on the device
    fe *data;                                // the bytes on the device; nullptr without any
};
int col_table(const std::vector<PolyBuf *> &cols, const void *data, size_t bytes, cudaStream_t s, ColTable *t);
int shared_poly_free(uint64_t h);            // h2_poly_free of a handle that is not the calling context's
// f(FpParams{}) or f(FqParams{}) for a field id; any other id fails
template <class F> static int by_field(int field, F &&f) {
    if (field == H2_FIELD_FP) return f(FpParams{});
    if (field == H2_FIELD_FQ) return f(FqParams{});
    return fail("unknown field id");
}
// f(FpParams{}, FqParams{}) for Pallas, f(FqParams{}, FpParams{}) for Vesta: (base field, scalar field); any other id fails
template <class F> static int by_curve(int curve, F &&f) {
    if (curve == H2_CURVE_PALLAS) return f(FpParams{}, FqParams{});
    if (curve == H2_CURVE_VESTA) return f(FqParams{}, FpParams{});
    return fail("unknown curve id");
}
static inline int check_curve(int curve) { return by_curve(curve, [](auto, auto) { return 0; }); }   // for entry points that check up front

// ---- functions one TU defines and others call -------------------------------------------------------------------
// Arrival of a one-shot MSM's inputs in k chunks: events on the copy stream -- bases / scalars of chunk j have landed.
// When the inputs are staged from pageable memory an uploader thread records the events while the calling thread issues
// the kernels: `recorded` (2 j + 1 after the scalars of chunk j, 2 j + 2 after its bases) tells the issuer that an event
// HAS been recorded and may be waited on; `failed` aborts the issue.
struct BasesChunks {
    uint32_t k = 0;
    cudaEvent_t ev[H2_MAX_UPLOAD_CHUNKS], ev_scal[H2_MAX_UPLOAD_CHUNKS];
    std::atomic<uint32_t> *recorded = nullptr;
    std::atomic<int> *failed = nullptr;
    int wait_recorded(uint32_t want) const {
        if (!recorded) return 0;
        while (recorded->load(std::memory_order_acquire) < want) {
            if (failed && failed->load()) return 1;
            std::this_thread::yield();
        }
        return 0;
    }
};
// capi_msm.cu
int convert_points(int curve, affine *d, size_t n, int to_mont, cudaStream_t s);
// capi_ntt.cu
int get_twiddles_any(int field, const fe &omega_mont, uint32_t log_n, cudaStream_t s, const fe **out);
int convert_field(int field, fe *d, size_t n, int to_mont, cudaStream_t s);
