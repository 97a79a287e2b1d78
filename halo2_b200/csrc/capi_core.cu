// C ABI of the engine (include/halo2_b200.h), part 1 of 5: context, device binding, settings, test hooks, utilities.
#include "util_kernels.cuh"

#include <algorithm>

static thread_local std::string g_err;
int fail(const std::string &m) { g_err = m; return 1; }
const std::string &last_error_string() { return g_err; }
// Global because a release of a shared window table must invalidate the graphs of every lane; a lane that grows its own
// scratch invalidates the others' graphs too, which costs one re-capture each and nothing else.
std::atomic<uint64_t> g_alloc_gen{0};
Context g_ctxs[H2_MAX_DEVICES];
Context g_lanes[H2_MAX_LANES];
Context g_dead;
Context *g_primary = &g_ctxs[0];
thread_local Context *g_cur = nullptr;
thread_local uint64_t g_cur_epoch = 0;
std::atomic<uint64_t> g_epoch{0};
std::vector<int> g_multi;                // devices of the multi-GPU entry points (h2_multi_init), primary first
std::mutex g_life_mu, g_reg_mu;
static std::atomic<uint64_t> g_next_handle{1};
uint64_t new_handle() { return g_next_handle.fetch_add(1); }

// ---- lanes ----------------------------------------------------------------------------------------------------------
// Slot i of the table is g_lanes[i]: handle 0 = free.  binds counts the host threads bound to the lane.  Both under g_reg_mu.
struct LaneSlot { uint64_t handle = 0; uint32_t binds = 0; };
static LaneSlot g_lane_slots[H2_MAX_LANES];
// The calling thread's binding; a thread that exits while bound gives its binding back.
struct LaneBinding {
    int slot = -1; uint64_t handle = 0, epoch = 0;
    void drop() {   // under g_reg_mu
        if (slot >= 0 && epoch == g_epoch.load() && g_lane_slots[slot].handle == handle) g_lane_slots[slot].binds--;
        slot = -1; handle = 0;
    }
    ~LaneBinding() {
        if (slot < 0) return;
        std::lock_guard<std::mutex> lk(g_reg_mu);
        drop();
    }
};
static thread_local LaneBinding g_binding;
bool on_lane() { return g_binding.slot >= 0; }

// Objects every lane reads -- base sets and shared polynomials -- count the calls in flight that hold them (users, under
// g_reg_mu).  Their release takes them out of the registry first, so no new call finds them, then waits here.
static std::condition_variable g_users_cv;   // a shared object's users dropped to 0
static void user_drop(uint32_t &users) {     // under g_reg_mu
    if (--users == 0) g_users_cv.notify_all();
}
// The object is out of its registry: wait for the calls that hold it, then for the device, which covers the asynchronous
// reads those calls queued on any lane's stream.  Returns with g_reg_mu released; the caller frees the object.
static void wait_unused(std::unique_lock<std::mutex> &lk, const uint32_t &users) {
    g_users_cv.wait(lk, [&users] { return users == 0; });
    const int dev = g_primary->device;
    lk.unlock();
    cudaSetDevice(dev);
    cudaDeviceSynchronize();
}

std::map<uint64_t, BaseSet *> g_bases;
BasesRef::BasesRef(uint64_t handle, bool open_session) {
    std::lock_guard<std::mutex> lk(g_reg_mu);
    auto it = g_bases.find(handle);
    if (it == g_bases.end()) return;
    b = it->second;
    b->users++;
    if (open_session) b->sessions++;
}
BasesRef::~BasesRef() {
    if (!b) return;
    std::lock_guard<std::mutex> lk(g_reg_mu);
    user_drop(b->users);
}
void bases_session_end(uint64_t handle) {
    std::lock_guard<std::mutex> lk(g_reg_mu);
    auto it = g_bases.find(handle);
    if (it != g_bases.end() && it->second->sessions) it->second->sessions--;
}
static void bases_free(BaseSet *b) { b->buf.release(); b->table.release(); b->dtable.release(); delete b; }
// Waits for the calls on any lane that are reading the set; refuses while an open IPA session on any lane refers to it.
extern "C" int h2_bases_release(uint64_t handle) {
    std::unique_lock<std::mutex> lk(g_reg_mu);
    auto it = g_bases.find(handle);
    if (it == g_bases.end()) return fail("h2_bases_release: unknown handle");
    BaseSet *b = it->second;
    if (b->sessions) return fail("h2_bases_release: an open IPA session uses the base set (h2_ipa_finish it first)");
    g_bases.erase(it);                   // no new user finds it
    wait_unused(lk, b->users);
    bases_free(b);
    return 0;
}

std::map<uint64_t, PolyBuf *> g_shared_polys;
PolyBuf *PolyArgs::fits(PolyBuf *p, uint64_t len, const char *len_name) {
    if (!field_given && field < 0) field = p->field;
    if (p->field != field) {
        fail(who + (field_given ? ": the polynomial is not over the curve's scalar field" : ": the polynomials live in different fields"));
        return nullptr;
    }
    if (p->len < len) { fail(who + ": a polynomial holds fewer than " + len_name + " elements"); return nullptr; }
    return p;
}
PolyBuf *PolyArgs::out(uint64_t h, uint64_t len, const char *len_name) {
    auto it = g_ctx.polys.find(h);
    if (it == g_ctx.polys.end()) {
        bool shared;
        {
            std::lock_guard<std::mutex> lk(g_reg_mu);
            shared = g_shared_polys.count(h) != 0;
        }
        fail(who + (shared ? ": the polynomial is shared (read-only)" : ": unknown polynomial handle"));
        return nullptr;
    }
    outs.push_back(it->second);
    return fits(it->second, len, len_name);
}
PolyBuf *PolyArgs::in(uint64_t h, uint64_t len, const char *len_name) {
    auto it = g_ctx.polys.find(h);
    PolyBuf *p = it != g_ctx.polys.end() ? it->second : nullptr;
    if (!p) {
        std::lock_guard<std::mutex> lk(g_reg_mu);
        auto s = g_shared_polys.find(h);
        if (s != g_shared_polys.end()) {
            p = s->second;
            p->users++;
            held.push_back(p);
        }
    }
    if (!p) { fail(who + ": unknown polynomial handle"); return nullptr; }
    ins.push_back(p);
    return fits(p, len, len_name);
}
int PolyArgs::out(const uint64_t *h, size_t n, uint64_t len, const char *len_name, std::vector<PolyBuf *> &v) {
    v.resize(n);
    for (size_t i = 0; i < n; i++)
        if (!(v[i] = out(h[i], len, len_name))) return 1;
    return 0;
}
int PolyArgs::in(const uint64_t *h, size_t n, uint64_t len, const char *len_name, std::vector<PolyBuf *> &v) {
    v.resize(n);
    for (size_t i = 0; i < n; i++)
        if (!(v[i] = in(h[i], len, len_name))) return 1;
    return 0;
}
// Batch slices and product columns run concurrently: an output written twice, or read as another one's input, would race.
int PolyArgs::distinct(const char *role) {
    std::vector<PolyBuf *> so(outs), si(ins);
    std::sort(so.begin(), so.end());
    std::sort(si.begin(), si.end());
    if (std::adjacent_find(so.begin(), so.end()) != so.end()) return fail(who + ": " + role + " handle appears twice");
    for (PolyBuf *p : so)
        if (std::binary_search(si.begin(), si.end(), p)) return fail(who + ": " + role + " handle is also an input");
    return 0;
}
PolyArgs::~PolyArgs() {
    if (held.empty()) return;
    std::lock_guard<std::mutex> lk(g_reg_mu);
    for (PolyBuf *p : held) user_drop(p->users);
}
// From any thread and any context: the caller holds no Context mutex.
int shared_poly_free(uint64_t h) {
    std::unique_lock<std::mutex> lk(g_reg_mu);
    auto it = g_shared_polys.find(h);
    if (it == g_shared_polys.end()) return fail("h2_poly_free: unknown handle");
    PolyBuf *p = it->second;
    g_shared_polys.erase(it);            // no new user finds it
    wait_unused(lk, p->users);
    p->buf.release();
    delete p;
    return 0;
}

std::atomic<bool> g_prof_on{false};
std::vector<ProfSpan> g_prof;
// primary-context work only: lanes (and the secondary devices of a multi-GPU call) run on other threads
void prof_begin(int kind, cudaStream_t s) {
    if (!g_prof_on || &g_ctx != g_primary) return;
    ProfSpan sp; sp.kind = kind;
    cudaEventCreate(&sp.e0); cudaEventCreate(&sp.e1);
    cudaEventRecord(sp.e0, s);
    g_prof.push_back(sp);
}
void prof_end(cudaStream_t s) {
    if (!g_prof_on || g_prof.empty() || &g_ctx != g_primary) return;
    cudaEventRecord(g_prof.back().e1, s);
}
std::atomic<uint64_t> g_launches{0};

// ------------------------------------------------------------------------------------------------
// staged transfers for pageable caller memory
// ------------------------------------------------------------------------------------------------
#include <condition_variable>
#include <thread>
#include <immintrin.h>
namespace {
// Slice copy of the staging pool.  The destination (a pinned ring slot on upload) is written once and next read by the DMA
// engine, never by this core: non-temporal stores skip the read-for-ownership of every destination line (2 instead of 3
// bytes of DRAM traffic per byte copied) and leave the caches to the source.  Falls back to memcpy without AVX2.
__attribute__((target("avx2"))) static void copy_stream_avx2(uint8_t *d, const uint8_t *s, size_t n) {
    while (n && ((uintptr_t)d & 31u)) { *d++ = *s++; n--; }
    size_t v = n / 128;
    for (; v; v--, d += 128, s += 128) {
        __m256i a = _mm256_loadu_si256((const __m256i *)s), b = _mm256_loadu_si256((const __m256i *)(s + 32));
        __m256i c = _mm256_loadu_si256((const __m256i *)(s + 64)), e = _mm256_loadu_si256((const __m256i *)(s + 96));
        _mm256_stream_si256((__m256i *)d, a); _mm256_stream_si256((__m256i *)(d + 32), b);
        _mm256_stream_si256((__m256i *)(d + 64), c); _mm256_stream_si256((__m256i *)(d + 96), e);
    }
    n &= 127;
    if (n) memcpy(d, s, n);
    _mm_sfence();
}
std::atomic<int> g_copy_nt{1};
static void slice_copy(uint8_t *d, const uint8_t *s, size_t n) {
    static const bool avx2 = __builtin_cpu_supports("avx2");
    if (avx2 && g_copy_nt.load(std::memory_order_relaxed) && n >= 4096) copy_stream_avx2(d, s, n);
    else memcpy(d, s, n);
}
struct CopyPool {            // a handful of host threads that copy slices in parallel
    std::mutex mu;
    std::condition_variable cv, cv_done;
    std::vector<std::thread> threads;
    uint8_t *dst = nullptr; const uint8_t *src = nullptr; size_t bytes = 0;
    uint32_t parts = 0, next_part = 0, done_parts = 0; uint64_t job = 0;
    bool stop = false;
    uint32_t active = 0;     // workers a job is cut for (<= threads.size()): h2_test_set_copy_threads
    size_t part_lo(uint32_t p) const { return p >= parts ? bytes : (bytes / parts * p) & ~(size_t)127; }   // 128-byte aligned cuts
    void start(unsigned n) {
        active = n;
        for (unsigned i = 0; i < n; i++) threads.emplace_back([this] { run(); });
    }
    void run() {
        uint64_t seen = 0;
        std::unique_lock<std::mutex> lk(mu);
        for (;;) {
            cv.wait(lk, [&] { return stop || (job != seen && next_part < parts); });
            if (stop) return;
            const uint64_t my_job = job;
            while (next_part < parts && job == my_job) {
                const uint32_t p = next_part++;
                const size_t lo = part_lo(p), hi = part_lo(p + 1);
                uint8_t *d = dst; const uint8_t *s = src;
                lk.unlock();
                slice_copy(d + lo, s + lo, hi - lo);
                lk.lock();
                if (++done_parts == parts) cv_done.notify_all();
            }
            seen = my_job;
        }
    }
    // one job at a time (callers serialise on job_mu); the calling thread takes slices too
    std::mutex job_mu;
    void copy(void *d, const void *s, size_t n) {
        if (n < (1u << 20) || threads.empty() || active == 0) { slice_copy((uint8_t *)d, (const uint8_t *)s, n); return; }
        std::lock_guard<std::mutex> jl(job_mu);
        std::unique_lock<std::mutex> lk(mu);
        dst = (uint8_t *)d; src = (const uint8_t *)s; bytes = n;
        parts = (active < threads.size() ? active : (uint32_t)threads.size()) + 1; next_part = 0; done_parts = 0; job++;
        cv.notify_all();
        while (next_part < parts) {
            const uint32_t p = next_part++;
            const size_t lo = part_lo(p), hi = part_lo(p + 1);
            lk.unlock();
            slice_copy(dst + lo, src + lo, hi - lo);
            lk.lock();
            ++done_parts;
        }
        cv_done.wait(lk, [&] { return done_parts == parts; });
    }
    ~CopyPool() {
        { std::lock_guard<std::mutex> lk(mu); stop = true; }
        cv.notify_all();
        for (auto &t : threads) t.join();
    }
};
CopyPool *copy_pool() {
    static CopyPool *P = [] {
        CopyPool *p = new CopyPool();    // leaked on purpose: worker threads must not be joined from a static destructor
        unsigned hw = std::thread::hardware_concurrency();
        p->start(hw >= 64 ? 31 : hw >= 16 ? 7 : hw >= 4 ? 3 : 0);
        if (const char *e = getenv("H2_COPY_THREADS")) { long v = atol(e); if (v >= 0 && v <= 31) p->active = (uint32_t)v; }
        else p->active = hw >= 64 ? 15 : p->active;
        return p;
    }();
    return P;
}
std::atomic<int> g_staging{1};
}  // namespace
void h2_set_staging(int on) { g_staging.store(on ? 1 : 0); }
extern "C" int h2_test_set_staging(int on) { h2_set_staging(on); return 0; }
// staging-copy tuning (bench sweep): worker threads a copy is cut for (the caller's thread takes a slice too), NT stores on/off
extern "C" int h2_test_set_copy_threads(int n, int nt_stores) {
    CopyPool *P = copy_pool();
    std::lock_guard<std::mutex> jl(P->job_mu);
    if (n >= 0) P->active = (uint32_t)n < P->threads.size() ? (uint32_t)n : (uint32_t)P->threads.size();
    if (nt_stores >= 0) g_copy_nt.store(nt_stores ? 1 : 0);
    return 0;
}

int StageRing::ensure() {
    if (slot_bytes) return 0;
    const size_t sb = 8u << 20;
    for (int i = 0; i < SLOTS; i++) {
        CU(cudaHostAlloc((void **)&slot[i], sb, cudaHostAllocDefault));
        CU(cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming));
        busy[i] = false;
    }
    slot_bytes = sb;
    return 0;
}
void StageRing::destroy() {
    if (!slot_bytes) return;
    for (int i = 0; i < SLOTS; i++) { cudaFreeHost(slot[i]); cudaEventDestroy(done[i]); slot[i] = nullptr; }
    slot_bytes = 0;
}
static bool host_is_pageable(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}
int upload_async(void *d_dst, const void *h_src, size_t bytes, cudaStream_t s) {
    if (bytes == 0) return 0;
    if (bytes < (256u << 10) || !g_staging.load() || !host_is_pageable(h_src)) {
        CU(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, s));
        return 0;
    }
    StageRing &R = g_ctx.stage;
    if (R.ensure()) return 1;
    CopyPool *P = copy_pool();
    for (size_t off = 0; off < bytes; off += R.slot_bytes) {
        const size_t len = bytes - off < R.slot_bytes ? bytes - off : R.slot_bytes;
        const uint32_t i = R.next++ % StageRing::SLOTS;
        if (R.busy[i]) CU(cudaEventSynchronize(R.done[i]));
        P->copy(R.slot[i], (const uint8_t *)h_src + off, len);
        CU(cudaMemcpyAsync((uint8_t *)d_dst + off, R.slot[i], len, cudaMemcpyHostToDevice, s));
        CU(cudaEventRecord(R.done[i], s));
        R.busy[i] = true;
    }
    return 0;
}
int download_sync(void *h_dst, const void *d_src, size_t bytes, cudaStream_t s) {
    if (bytes == 0) { CU(cudaStreamSynchronize(s)); return 0; }
    if (bytes < (256u << 10) || !g_staging.load() || !host_is_pageable(h_dst)) {
        CU(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        return 0;
    }
    StageRing &R = g_ctx.stage;
    if (R.ensure()) return 1;
    CopyPool *P = copy_pool();
    // DMA into the slots round-robin; a slot is drained into the caller's buffer before it is reused
    struct Pending { uint32_t slot; size_t off, len; };
    std::vector<Pending> q;
    size_t head = 0;
    auto drain = [&](const Pending &e) -> int {
        CU(cudaEventSynchronize(R.done[e.slot]));
        P->copy((uint8_t *)h_dst + e.off, R.slot[e.slot], e.len);
        R.busy[e.slot] = false;
        return 0;
    };
    for (size_t off = 0; off < bytes; off += R.slot_bytes) {
        const size_t len = bytes - off < R.slot_bytes ? bytes - off : R.slot_bytes;
        const uint32_t i = R.next++ % StageRing::SLOTS;
        while (head < q.size() && q[head].slot == i) { if (drain(q[head])) return 1; head++; }
        if (R.busy[i]) CU(cudaEventSynchronize(R.done[i]));     // an upload still in flight from this slot
        CU(cudaMemcpyAsync(R.slot[i], (const uint8_t *)d_src + off, len, cudaMemcpyDeviceToHost, s));
        CU(cudaEventRecord(R.done[i], s));
        R.busy[i] = true;
        q.push_back({i, off, len});
    }
    for (; head < q.size(); head++) if (drain(q[head])) return 1;
    return 0;
}

int require_ready() {
    if (&g_ctx == &g_dead) return fail("the lane this thread was bound to was destroyed by h2_shutdown: bind another (h2_lane_bind, 0 = the primary context)");
    if (!g_ctx.ready) return fail("h2_init has not been called (or failed): no CUDA device bound; there is no CPU fallback");
    CU(cudaSetDevice(g_ctx.device));
    return 0;
}
int scratch_acquire(cudaStream_t s) {
    if (g_ctx.have_last) CU(cudaStreamWaitEvent(s, g_ctx.last_use, 0));
    return 0;
}
int scratch_release(cudaStream_t s) {
    CU(cudaEventRecord(g_ctx.last_use, s));
    g_ctx.have_last = true;
    return 0;
}

extern "C" const char *h2_last_error(void) { return g_err.c_str(); }
extern "C" uint32_t h2_abi_version(void) { return 1; }
extern "C" uint64_t h2_launch_count(void) { return g_launches.load(); }
extern "C" int h2_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}
static int ctx_create(Context &C, int device) {
    CU(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail("h2_init: this library is built for sm_90a (H100) only");
    CU(cudaStreamCreateWithFlags(&C.stream, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&C.last_use, cudaEventDisableTiming));
    CU(cudaStreamCreateWithFlags(&C.copy_stream, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&C.ev_scalars_up, cudaEventDisableTiming));
    for (int j = 0; j < H2_MAX_UPLOAD_CHUNKS; j++) {
        CU(cudaEventCreateWithFlags(&C.ev_bases_up[j], cudaEventDisableTiming));
        CU(cudaEventCreateWithFlags(&C.ev_scal_up[j], cudaEventDisableTiming));
    }
    C.device = device;
    C.ready = true;
    return 0;
}
static void ctx_destroy(Context &C) {
    if (!C.ready) return;
    cudaSetDevice(C.device);
    cudaDeviceSynchronize();
    DevBuf *all[] = {&C.scal_in, &C.bases_in, &C.bases_phi, &C.glv_parts, &C.scal_canon, &C.counts, &C.cursor, &C.refs, &C.size_hist,
                     &C.items, &C.bucket_sum, &C.pkey, &C.pstart, &C.pend, &C.ppt, &C.ra_t, &C.ra_e,
                     &C.r0, &C.r1, &C.wsum, &C.scan_blocks, &C.result, &C.misc, &C.ntt_io, &C.ntt_out,
                     &C.ntt_work, &C.pow2, &C.ec_work, &C.ec_io, &C.ec_out, &C.fb_a, &C.fb_b, &C.po_lvl, &C.po_q, &C.po_pts, &C.po_ptrs, &C.ast_code, &C.ast_consts,
                     &C.multi_parts, &C.ba_lv[0], &C.ba_lv[1], &C.ba_lv[2], &C.lk_keys, &C.lk_aux, &C.lk_u32, &C.kg_tab, &C.kg_map,
                     &C.as_edge, &C.as_cell, &C.as_slot, &C.gp_val, &C.gp_aux};
    for (DevBuf *b : all) b->release();
    for (auto *t : C.twiddles) { t->buf.release(); delete t; }
    C.twiddles.clear();
    for (auto &kv : C.shards) bases_free(kv.second);
    C.shards.clear();
    for (auto &kv : C.ipa) {
        IpaSession *q = kv.second;
        bases_session_end(q->bases);
        q->p.release(); q->b.release(); q->s.release(); q->scal.release(); q->out.release(); delete q;
    }
    C.ipa.clear();
    for (auto &kv : C.polys) { kv.second->buf.release(); delete kv.second; }
    C.polys.clear();
    for (PolyBuf *q : C.poly_pool) { q->buf.release(); delete q; }
    C.poly_pool.clear();
    for (auto &ge : C.graphs) if (ge.exec) cudaGraphExecDestroy(ge.exec);
    C.graphs.clear();
    for (IpaSession *q : C.ipa_pool) { q->p.release(); q->b.release(); q->s.release(); q->scal.release(); q->out.release(); delete q; }
    C.ipa_pool.clear();
    C.stage.destroy();
    if (C.h_flags) { cudaFreeHost(C.h_flags); C.h_flags = nullptr; }
    cudaEventDestroy(C.ev_scalars_up);
    for (int j = 0; j < H2_MAX_UPLOAD_CHUNKS; j++) { cudaEventDestroy(C.ev_bases_up[j]); cudaEventDestroy(C.ev_scal_up[j]); }
    cudaStreamDestroy(C.copy_stream);
    cudaEventDestroy(C.last_use);
    cudaStreamDestroy(C.stream);
    C = Context();
}
extern "C" int h2_init(int device) {
    std::lock_guard<std::mutex> life(g_life_mu);
    if (g_primary->ready && g_primary->device == device) return 0;
    if (g_primary->ready) return fail("h2_init: already bound to another device (one process per GPU; h2_multi_init adds devices)");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) return fail(std::string("h2_init: no CUDA device: ") + cudaGetErrorString(e));
    if (device < 0 || device >= n || device >= H2_MAX_DEVICES) return fail("h2_init: device index out of range");
    {
        std::lock_guard<std::mutex> lk(g_ctxs[device].mu.m);
        if (ctx_create(g_ctxs[device], device)) { ctx_destroy(g_ctxs[device]); return 1; }
    }
    std::lock_guard<std::mutex> reg(g_reg_mu);
    g_primary = &g_ctxs[device];
    return 0;
}
// Single-process multi-GPU (SURVEY.md section 8(b): a Rust caller of best_multiexp is ONE process): binds contexts to
// `ngpu` devices -- the primary one first, then the others in index order -- and enables peer access to the primary.
// The h2_multi_* calls run on the primary context only: a thread bound to a lane is refused.
extern "C" int h2_multi_init(int ngpu) {
    if (on_lane()) return fail("h2_multi_init: the multi-GPU entry points run on the primary context, not on a lane (h2_lane_bind(0))");
    std::lock_guard<std::mutex> life(g_life_mu);
    CtxLock lk;
    if (require_ready()) return 1;
    int n = 0;
    CU(cudaGetDeviceCount(&n));
    if (ngpu < 1 || ngpu > n || ngpu > H2_MAX_DEVICES) return fail("h2_multi_init: ngpu out of range (" + std::to_string(n) + " devices visible)");
    const int prim = g_primary->device;
    std::vector<int> devs{prim};
    for (int d = 0; d < n && (int)devs.size() < ngpu; d++) if (d != prim) devs.push_back(d);
    for (int d : devs) {
        if (g_ctxs[d].ready) continue;
        if (ctx_create(g_ctxs[d], d)) { ctx_destroy(g_ctxs[d]); cudaSetDevice(prim); return 1; }
        // settings follow the primary context
        g_ctxs[d].glv_on = g_primary->glv_on; g_ctxs[d].sort_bins = g_primary->sort_bins; g_ctxs[d].window_override = g_primary->window_override;
        g_ctxs[d].chunk_min_log = g_primary->chunk_min_log;
        int can = 0;
        if (cudaDeviceCanAccessPeer(&can, d, prim) == cudaSuccess && can) { cudaSetDevice(d); if (cudaDeviceEnablePeerAccess(prim, 0) != cudaSuccess) cudaGetLastError(); }
        if (cudaDeviceCanAccessPeer(&can, prim, d) == cudaSuccess && can) { cudaSetDevice(prim); if (cudaDeviceEnablePeerAccess(d, 0) != cudaSuccess) cudaGetLastError(); }
    }
    CU(cudaSetDevice(prim));
    std::lock_guard<std::mutex> reg(g_reg_mu);
    g_multi = devs;
    return 0;
}
extern "C" int h2_multi_count(void) {
    std::lock_guard<std::mutex> reg(g_reg_mu);
    return (int)g_multi.size();
}
void multi_bases_clear();   // capi_msm.cu
extern "C" int h2_shutdown(void) {
    std::lock_guard<std::mutex> life(g_life_mu);
    // every context's mutex: calls in flight on any lane finish first
    std::vector<std::unique_lock<std::mutex>> held;
    held.emplace_back(g_primary->mu.m);
    std::vector<int> live;
    {
        std::lock_guard<std::mutex> reg(g_reg_mu);
        for (int i = 0; i < H2_MAX_LANES; i++) if (g_lane_slots[i].handle) live.push_back(i);
    }
    for (int i : live) held.emplace_back(g_lanes[i].mu.m);
    {   // from here on no lane handle is known and every thread bound to one finds its lane gone
        std::lock_guard<std::mutex> reg(g_reg_mu);
        for (auto &s : g_lane_slots) s = LaneSlot();
        g_binding.slot = -1; g_binding.handle = 0;
        g_epoch++;
    }
    for (int i : live) ctx_destroy(g_lanes[i]);
    for (int d = 0; d < H2_MAX_DEVICES; d++) ctx_destroy(g_ctxs[d]);
    set_cur(nullptr);
    std::lock_guard<std::mutex> reg(g_reg_mu);
    for (auto &kv : g_bases) bases_free(kv.second);
    g_bases.clear();
    for (auto &kv : g_shared_polys) { kv.second->buf.release(); delete kv.second; }   // every context is idle and synchronised
    g_shared_polys.clear();
    multi_bases_clear();
    g_multi.clear();
    g_primary = &g_ctxs[0];
    return 0;
}

// A lane: one more Context on the primary device (ctx.cuh), for one prover thread.  It starts with the library's default
// settings and owns what is created on it.
extern "C" int h2_lane_create(uint64_t *lane) {
    std::lock_guard<std::mutex> life(g_life_mu);
    if (!g_primary->ready) return fail("h2_lane_create: h2_init has not been called (or failed)");
    int slot = -1;
    {
        std::lock_guard<std::mutex> reg(g_reg_mu);
        for (int i = 0; i < H2_MAX_LANES && slot < 0; i++) if (!g_lane_slots[i].handle) slot = i;
    }
    if (slot < 0) return fail("h2_lane_create: all " + std::to_string(H2_MAX_LANES) + " lanes are in use (h2_lane_destroy one)");
    Context &L = g_lanes[slot];
    {
        std::lock_guard<std::mutex> lk(L.mu.m);
        if (ctx_create(L, g_primary->device)) { ctx_destroy(L); return 1; }
    }
    std::lock_guard<std::mutex> reg(g_reg_mu);
    g_lane_slots[slot].handle = new_handle();
    g_lane_slots[slot].binds = 0;
    *lane = g_lane_slots[slot].handle;
    return 0;
}
// Binds the calling host thread to `lane` (0: the primary context): every later call from this thread runs there.
extern "C" int h2_lane_bind(uint64_t lane) {
    std::lock_guard<std::mutex> reg(g_reg_mu);
    int slot = -1;
    if (lane) {
        for (int i = 0; i < H2_MAX_LANES && slot < 0; i++) if (g_lane_slots[i].handle == lane) slot = i;
        if (slot < 0) return fail("h2_lane_bind: unknown lane handle");
    }
    g_binding.drop();
    if (slot < 0) { set_cur(nullptr); return 0; }
    g_lane_slots[slot].binds++;
    g_binding.slot = slot; g_binding.handle = lane; g_binding.epoch = g_epoch.load();
    set_cur(&g_lanes[slot]);
    return 0;
}
// Frees the lane's polynomials, IPA sessions, pools and streams.  Refused while another thread is bound to it; the calling
// thread, if bound to it, goes back to the primary context.
extern "C" int h2_lane_destroy(uint64_t lane) {
    std::lock_guard<std::mutex> life(g_life_mu);
    int slot = -1;
    {
        std::lock_guard<std::mutex> reg(g_reg_mu);
        for (int i = 0; i < H2_MAX_LANES && slot < 0; i++) if (lane && g_lane_slots[i].handle == lane) slot = i;
        if (slot < 0) return fail("h2_lane_destroy: unknown lane handle");
        const bool mine = g_binding.slot == slot;
        if (g_lane_slots[slot].binds > (mine ? 1u : 0u)) return fail("h2_lane_destroy: another thread is bound to the lane");
        if (mine) { g_binding.drop(); set_cur(nullptr); }
        g_lane_slots[slot] = LaneSlot();   // unknown from here on: nobody can bind it
    }
    std::lock_guard<std::mutex> lk(g_lanes[slot].mu.m);
    ctx_destroy(g_lanes[slot]);
    return 0;
}

extern "C" int h2_set_glv(int on) {
    CtxLock lk;
    g_ctx.glv_on = on ? 1u : 0u;
    return 0;
}
extern "C" int h2_set_sort_mode(int exact_only) {
    CtxLock lk;
    g_ctx.sort_bins = exact_only ? 0u : 1u;
    return 0;
}
// test hook: flags of the most recent MSM -- bit 0: some bucket was split into several work items, bit 1: the exact
// sort ran (bin overflow, or no bins).  Synchronises the device.
extern "C" int h2_test_last_msm_flags(uint32_t *out) {
    CtxLock lk;
    if (require_ready()) return 1;
    if (!g_ctx.last_flags) return fail("h2_test_last_msm_flags: no MSM has run");
    uint32_t f[2];
    CU(cudaDeviceSynchronize());
    CU(cudaMemcpyAsync(f, g_ctx.last_flags, sizeof f, cudaMemcpyDeviceToHost, g_ctx.stream));   // not on the legacy default stream
    CU(cudaStreamSynchronize(g_ctx.stream));
    *out = (f[0] ? 1u : 0u) | (f[1] ? 2u : 0u);
    return 0;
}
// test hook: what the most recent MSM pass ran (recorded on the host by msm_run; layout in include/halo2_b200.h)
extern "C" int h2_test_last_msm_plan(uint32_t out[8]) {
    CtxLock lk;
    if (require_ready()) return 1;
    if (!g_ctx.have_plan) return fail("h2_test_last_msm_plan: no MSM has run");
    memcpy(out, g_ctx.last_plan, sizeof g_ctx.last_plan);
    return 0;
}
// The settings hooks below act on the calling thread's lane; on the primary context they act on every device's context,
// so that the multi-GPU workers follow.
static void for_settings(const std::function<void(Context &)> &f) {
    if (on_lane()) { f(g_ctx); return; }
    for (int d = 0; d < H2_MAX_DEVICES; d++) f(g_ctxs[d]);
}
// test / A-B hook: fixed-base passes first run without their fallback kernels (1, default) or always run the full pass (0)
extern "C" int h2_test_set_fast_fixed(int on) {
    CtxLock lk;
    // on > 1 (tuning): log2 of the bucket count up to which a fast pass takes its buckets in index order (on = 2: never)
    for_settings([on](Context &C) { C.fast_on = on ? 1u : 0u; if (on > 1) C.natural_max_buckets = on == 2 ? 0 : 1ull << on; });
    return 0;
}
// test hook: small polynomials reduce in one CTA each (1, default) or through the level tree like large ones (0)
extern "C" int h2_test_set_poly_cta(int on) {
    CtxLock lk;
    for_settings([on](Context &C) { C.poly_cta = on ? 1u : 0u; });
    return 0;
}
// test hook: CUDA-graph replay of fixed-base MSMs on / off
extern "C" int h2_test_set_graphs(int on) {
    CtxLock lk;
    g_ctx.graphs_on = on ? 1u : 0u;
    return 0;
}
// test hook: quads per work item of the small-problem accumulation (1, 2 or 4).  Invalidates nothing: graphs are keyed by
// their parameters only, so flip it before the first fixed-base MSM of a base set or with graphs off.
extern "C" int h2_test_set_accum_ways(uint32_t ways) {
    CtxLock lk;
    if (ways >> 8) { g_ctx.small_accum_refs = 1ull << (ways >> 8); ways &= 0xffu; }   // tuning: bits 8.. = log2 of the reference count up to which lanes cooperate
    if (ways != 0 && ways != 1 && ways != 2 && ways != 4 && ways != 12 && ways != 14)
        return fail("h2_test_set_accum_ways: 0 (a pair of lanes), 1, 2 or 4 (quads), 12 / 14 (2 / 4 independent lanes per item)");
    g_ctx.accum_ways = ways;
    for (auto &ge : g_ctx.graphs) if (ge.exec) { cudaGraphExecDestroy(ge.exec); ge.exec = nullptr; ge.seen = 0; }
    return 0;
}
// test / tuning hook: batched-affine halving rounds ahead of the XYZZ accumulation of large one-shot MSMs (0 = classic
// accumulation only, at most 3) and the pairs per thread that share one inversion (0 keeps the current value)
extern "C" int h2_test_set_batched_affine(uint32_t rounds, uint32_t pairs_per_thread) {
    CtxLock lk;
    const uint32_t variant = rounds >> 8;     // bits 8..: kernel variant + 1 (tuning; 0 = the default variant)
    rounds &= 0xffu;
    if (rounds > H2_BA_MAX_ROUNDS) return fail("h2_test_set_batched_affine: at most 3 rounds");
    for_settings([=](Context &C) {
        C.ba_rounds = rounds; C.ba_variant = variant ? variant - 1 : 3;
        if (pairs_per_thread) C.ba_target = pairs_per_thread;
    });
    return 0;
}
// test hook: EC-FFT butterfly form -- 1: quads of lanes, 0: one thread each, -1: by size (the default)
extern "C" int h2_test_set_ecfft_quad(int on) {
    CtxLock lk;
    g_ctx.ecfft_quad = on < 0 ? 1u : on ? 2u : 0u;   // -1: by size (default), 0: thread form, 1: quad form
    return 0;
}
// test hook: one-shot MSMs (h2_msm) of >= 2^log2_n points upload their bases in chunks (default 19)
// tuning hook: where a k-chunk upload cuts its points, in sixteenths (k = 2 .. 4; c1 < c2 < c3 < 16, unused ones ignored)
extern uint32_t g_chunk_cut[H2_MAX_UPLOAD_CHUNKS + 1][H2_MAX_UPLOAD_CHUNKS + 1];
extern "C" int h2_test_set_chunk_cuts(uint32_t k, uint32_t c1, uint32_t c2, uint32_t c3) {
    CtxLock lk;
    if (k < 2 || k > H2_MAX_UPLOAD_CHUNKS) return fail("h2_test_set_chunk_cuts: k must be 2, 3 or 4");
    const uint32_t c[5] = {0, c1, k > 2 ? c2 : 16, k > 3 ? c3 : 16, 16};
    for (uint32_t j = 1; j <= 4; j++) if (c[j] < c[j - 1] || c[j] > 16 || (j < k && c[j] == c[j - 1])) return fail("h2_test_set_chunk_cuts: cuts must increase, below 16");
    for (uint32_t j = 0; j <= 4; j++) g_chunk_cut[k][j] = c[j];
    return 0;
}
extern "C" int h2_test_set_chunk_threshold(uint32_t log2_n) {
    CtxLock lk;
    if (log2_n > 40) return fail("h2_test_set_chunk_threshold: log2_n > 40");
    g_ctx.chunk_min_log = log2_n;
    return 0;
}
extern "C" int h2_set_window_bits(uint32_t c) {
    if (c > 24) return fail("h2_set_window_bits: c must be <= 24");
    CtxLock lk;
    g_ctx.window_override = c;
    return 0;
}

extern "C" int h2_dev_gen_points(int curve, uint64_t seed, uint64_t first, size_t n, void *d_out, void *stream) {
    CtxLock lk;
    if (require_ready()) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    return by_curve(curve, [&](auto p, auto) {
        if (n) LAUNCH(gen_points_kernel<decltype(p)>, blocks_for(n, 128), 128, 0, s, (affine *)d_out, seed, first, (uint64_t)n);
        return 0;
    });
}
extern "C" int h2_dev_convert(int field, void *d_a, size_t n, int to_montgomery, void *stream) {
    CtxLock lk;
    if (require_ready()) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return 0;
    return by_field(field, [&](auto p) {
        LAUNCH(convert_kernel<decltype(p)>, blocks_for(n, 256), 256, 0, s, (fe *)d_a, (uint64_t)n, to_montgomery);
        return 0;
    });
}
extern "C" int h2_test_field_op(int field, int op, const void *a, const void *b, size_t n, void *out) {
    CtxLock lk;
    if (require_ready()) return 1;
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (scratch_acquire(s)) return 1;
    if (X.misc.ensure(3 * n * sizeof(fe) + 64)) return 1;
    fe *da = X.misc.as<fe>(), *db = da + n, *dout = db + n;
    CU(cudaMemcpyAsync(da, a, n * sizeof(fe), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(db, b, n * sizeof(fe), cudaMemcpyHostToDevice, s));
    if (by_field(field, [&](auto p) {
            LAUNCH(test_field_kernel<decltype(p)>, blocks_for(n, 128), 128, 0, s, da, db, dout, (uint64_t)n, op);
            return 0;
        }))
        return 1;
    CU(cudaMemcpyAsync(out, dout, n * sizeof(fe), cudaMemcpyDeviceToHost, s));
    if (scratch_release(s)) return 1;
    CU(cudaStreamSynchronize(s));
    return 0;
}
extern "C" int h2_test_curve_op(int curve, int op, const void *a_xy, const void *b_xy, size_t n, void *out_xy) {
    CtxLock lk;
    if (op < 0 || op > 13)
        return fail("h2_test_curve_op: op must be 0 (mixed and full add), 1 (double), 2 (scalar mul), 3 .. 6 (xyzz_add, xyzz_add_mixed, "
                    "xyzz_double, xyzz_shift), 7 .. 10 (xyzz_add_quad, xyzz_add_mixed_quad, xyzz_add_mixed_pair, xyzz_shift_quad), "
                    "11 / 12 (xyzz_addsub_q sum / difference) or 13 (xyzz_double_q)");
    if (require_ready()) return 1;
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (scratch_acquire(s)) return 1;
    if (X.misc.ensure(3 * n * sizeof(affine) + 64)) return 1;
    affine *da = X.misc.as<affine>(), *db = da + n, *dout = db + n;
    CU(cudaMemcpyAsync(da, a_xy, n * sizeof(affine), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(db, b_xy, n * sizeof(affine), cudaMemcpyHostToDevice, s));
    if (by_curve(curve, [&](auto p, auto) {
            if (op <= 6) LAUNCH(test_curve_kernel<decltype(p)>, blocks_for(n, 64), 64, 0, s, da, db, dout, (uint64_t)n, op);
            else LAUNCH(test_curve_coop_kernel<decltype(p)>, blocks_for(n * (op == 9 ? 2 : 4), 64), 64, 0, s, da, db, dout, (uint64_t)n, op);   // whole warps
            return 0;
        }))
        return 1;
    CU(cudaMemcpyAsync(out_xy, dout, n * sizeof(affine), cudaMemcpyDeviceToHost, s));
    if (scratch_release(s)) return 1;
    CU(cudaStreamSynchronize(s));
    return 0;
}
extern "C" int h2_bench_field_mul(int field, uint32_t threads_per_block, uint32_t blocks, uint32_t iters, float *ms) {
    CtxLock lk;
    if (require_ready()) return 1;
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (scratch_acquire(s)) return 1;
    size_t threads = (size_t)threads_per_block * blocks;
    if (X.misc.ensure(threads * 4 * sizeof(fe))) return 1;
    CU(cudaMemsetAsync(X.misc.p, 0x11, threads * 4 * sizeof(fe), s));
    cudaEvent_t e0, e1;
    CU(cudaEventCreate(&e0)); CU(cudaEventCreate(&e1));
    for (int rep = 0; rep < 2; rep++) {   // first repetition warms up
        CU(cudaEventRecord(e0, s));
        // field | 0x100: the same loop with fe_sqr
        if (field == H2_FIELD_FP) LAUNCH((bench_mul_kernel<FpParams, false>), blocks, threads_per_block, 0, s, X.misc.as<fe>(), iters);
        else if (field == H2_FIELD_FQ) LAUNCH((bench_mul_kernel<FqParams, false>), blocks, threads_per_block, 0, s, X.misc.as<fe>(), iters);
        else if (field == (H2_FIELD_FP | 0x100)) LAUNCH((bench_mul_kernel<FpParams, true>), blocks, threads_per_block, 0, s, X.misc.as<fe>(), iters);
        else LAUNCH((bench_mul_kernel<FqParams, true>), blocks, threads_per_block, 0, s, X.misc.as<fe>(), iters);
        CU(cudaEventRecord(e1, s));
        CU(cudaStreamSynchronize(s));
    }
    CU(cudaEventElapsedTime(ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return scratch_release(s);
}

// mode: 0 dependent mul chain, 1 two chains, 2 four chains, 3 xyzz_double, 4 xyzz_add, 5 xyzz_add_mixed;
// one warp, `iters` iterations; *ms = elapsed.
extern "C" int h2_bench_latency(int mode, uint32_t iters, float *ms) {
    CtxLock lk;
    if (require_ready()) return 1;
    Context &X = g_ctx;
    cudaStream_t s = X.stream;
    if (scratch_acquire(s)) return 1;
    if (X.misc.ensure(32 * 4 * sizeof(fe))) return 1;
    CU(cudaMemsetAsync(X.misc.p, 0x11, 32 * 4 * sizeof(fe), s));
    cudaEvent_t e0, e1;
    CU(cudaEventCreate(&e0)); CU(cudaEventCreate(&e1));
    for (int rep = 0; rep < 2; rep++) {
        CU(cudaEventRecord(e0, s));
        LAUNCH(bench_latency_kernel<FpParams>, 1, 32, 0, s, X.misc.as<fe>(), iters, mode);
        CU(cudaEventRecord(e1, s));
        CU(cudaStreamSynchronize(s));
    }
    CU(cudaEventElapsedTime(ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return scratch_release(s);
}

// ------------------------------------------------------------------------------------------------
// per-kernel timing for the roofline leg of bench.py
// ------------------------------------------------------------------------------------------------
// The records (g_prof) are of primary-context work and guarded by the primary's mutex, whichever thread asks.
extern "C" int h2_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(g_primary->mu.m);
    if (require_ready()) return 1;
    cudaDeviceSynchronize();
    for (auto &sp : g_prof) { cudaEventDestroy(sp.e0); cudaEventDestroy(sp.e1); }
    g_prof.clear();
    g_prof_on = on != 0;
    return 0;
}
// kind 0 = msm_accum0_kernel, 1 = ntt_pass_kernel.  Returns summed device time and launch count.
extern "C" int h2_profile_read(int kind, float *total_ms, uint32_t *launches) {
    std::lock_guard<std::mutex> lk(g_primary->mu.m);
    if (require_ready()) return 1;
    CU(cudaDeviceSynchronize());
    float tot = 0; uint32_t cnt = 0;
    for (auto &sp : g_prof) {
        if (sp.kind != kind) continue;
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, sp.e0, sp.e1));
        tot += ms; cnt++;
    }
    *total_ms = tot; *launches = cnt;
    return 0;
}

