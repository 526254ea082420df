// libafcrypto.so — C-ABI layer (include/afcrypto.h) over the sm_90a kernels.
//
// Host-side responsibilities only: context + stream pool, pinned/device staging, chunked
// copy/compute overlap for host-buffer calls, the RFC 6962 level schedule, optional NCCL (dlopen).
// There is deliberately NO CPU implementation of any primitive in this library: if CUDA is missing or
// fails, calls return AFC_ECUDA and the reference-side adapter decides what to do (INTEGRATION.md).
#include "../../include/afcrypto.h"
#include "afc_internal.h"
#include "afc_launch.h"

#include <atomic>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>
#include <sched.h>
#include <mutex>
#include <string>
#include <vector>

using namespace afc;

namespace {

constexpr int kLanes = 4;                 // concurrent host-buffer calls per context
constexpr int kSlots = 4;                 // chunks in flight per call: copies keep streaming while an earlier chunk computes
constexpr uint32_t kChunkItems = 1u << 17;  // items per pipeline chunk for host-buffer calls (one full wave of the table-driven verify at G = 2)
constexpr size_t kChunkBytes = 96u << 20;   // and at most this many message bytes per chunk
constexpr uint32_t kMinChunkItems = 1u << 16;   // the tail of a call tapers down to this (fewer, larger copies than 16 k)

struct DevBuf {
    uint8_t* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 4 + 256;
        cudaError_t e = cudaMalloc((void**)&p, want);
        // zeroed once: the kernels read whole aligned words and mask what lies past a message, so the slack behind the last
        // staged byte is read (never used); this keeps those reads defined without a memset per call
        if (e == cudaSuccess) e = cudaMemset(p, 0, want);
        // the memset runs on the legacy default stream and returns before it has happened; the buffer's users are NON-BLOCKING
        // streams, which do not order themselves after it: without this wait a copy enqueued next could be zeroed afterwards
        // (seen once as a wrong Merkle root right after a log was created)
        if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
struct PinBuf {
    uint8_t* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t n, afc_ctx* ctx) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 4 + 256;
        p = (uint8_t*)afc_internal_pinned_alloc(ctx, want);        // on the NUMA node of the context's GPU
        if (!p) return cudaErrorMemoryAllocation;
        cap = want;
        return cudaSuccess;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

// One stage of a lane's ring of in-flight chunks
struct Slot {
    cudaStream_t stream = nullptr;
    DevBuf arena;                            // a chunk's staged inputs, outputs and scratch, carved per call
    PinBuf h_in, h_out;                      // bounce buffers for the caller's pageable memory: inputs, outputs
};
struct Lane {
    Slot slot[kSlots];
    bool busy = false;
};

}  // namespace

struct afc_ctx {
    int device = 0;
    cudaDeviceProp prop{};
    void* comb = nullptr;
    void* ct16 = nullptr;               // 48 KB constant-time signing table (radix 16), gathered from comb at init
    bool sign_ct = true;                // secret scalars go through the constant-time fixed-base multiplication (AFC_SIGN_CT=0: fast path)
    Lane lanes[kLanes];
    std::mutex mu;
    std::condition_variable cv;
    std::atomic<unsigned long long> launches{0};
    std::string last_error;
    // CPUs next to this GPU (sysfs local_cpulist of its PCI device): pinned staging is allocated from a thread bound to them
    cpu_set_t local_cpus;
    bool has_local_cpus = false;
    int numa_node = -1;
    // transparent issuer-key cache behind afc_ed25519_verify_batch (see k_ed25519.cu)
    launch::KeyCache kc{};
    bool kc_ready = false;
    uint32_t kc_max_keys = 4096;        // AFC_KEYCACHE_MAX_KEYS / afc_keycache_configure; 0 disables (4096 keys = 1.6 GB of an H100's 80 GB)
    uint32_t kc_call_cap = 0;           // per-call scratch capacity (items)
    std::mutex kc_mu;
    cudaEvent_t kc_event = nullptr;     // orders successive users of the cache across streams
    // per-kernel CUDA-event profiling (afc_profile_begin / afc_profile_end)
    bool profile = false;
    std::vector<launch::LaunchRec> prof_recs;
    int prof_next = 0;                  // claimed with __atomic_fetch_add (launch::LaunchLog::begin)
    // NCCL (lazy)
    void* nccl_lib = nullptr;
    void* nccl_comm = nullptr;
    int nranks = 0, rank = 0;
    cudaStream_t comm_stream = nullptr;
    uint8_t* d_comm_buf = nullptr;
};

struct afc_keyset {
    afc_ctx* ctx = nullptr;
    uint32_t n_keys = 0;
    uint8_t* d_pks = nullptr;      // n_keys x 32
    uint8_t* d_valid = nullptr;    // n_keys
    void* d_tabs = nullptr;        // n_keys x 32 x 128 ge_precomp
    size_t tab_bytes = 0;
    // afc_keyset_new_named: the keys' DIDs and an open-addressing table DID -> key index (FNV-1a, linear probing), plus the two
    // document schemas the stored-document call parses with (afc_vcdoc.cuh)
    bool named = false;
    uint8_t* d_dids = nullptr;     // DID bytes back to back
    uint32_t* d_did_off = nullptr; // n_keys + 1
    uint32_t* d_slots = nullptr;   // slot_mask + 1 entries, 0xffffffff = empty
    uint32_t slot_mask = 0;
    uint8_t* d_schemas = nullptr;  // 2 x launch::vc_schema_bytes(): execution VC, workflow VC
    uint8_t* d_vcj_schemas = nullptr;  // 2 x launch::vcj_schema_bytes(): the same for documents in any spelling (afc_vcjson.cuh)
};

struct afc_merkle_tree {
    afc_ctx* ctx = nullptr;
    uint64_t n = 0;
    std::vector<uint8_t*> levels;        // device pointers, level 0 = leaf hashes
    std::vector<uint64_t> sizes;
    uint8_t** d_levels = nullptr;        // the same table on the device
    uint64_t* d_sizes = nullptr;
};

struct afc_merkle {
    afc_ctx* ctx = nullptr;
    uint64_t size = 0;
    uint8_t* d_frontier = nullptr;   // 64 x 32
    uint8_t* d_root = nullptr;       // 32
    DevBuf lv[2], leaves, off;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev = nullptr;        // last device-side work enqueued on a caller's stream (orders _dev calls vs host calls)
    std::mutex mu;
};

namespace {

#define CK(expr)                                                           \
    do {                                                                   \
        cudaError_t _e = (expr);                                           \
        if (_e != cudaSuccess) { set_err(ctx, _e, #expr); return AFC_ECUDA; } \
    } while (0)

void set_err(afc_ctx* ctx, cudaError_t e, const char* what) {
    if (!ctx) return;
    std::lock_guard<std::mutex> g(ctx->mu);
    ctx->last_error = std::string(cudaGetErrorName(e)) + ": " + cudaGetErrorString(e) + " at " + what;
}

// Per-call launch log: counts launches; when profiling is on every launch claims one event pair from the ctx pool.
struct CallLog {
    afc_ctx* ctx;
    launch::LaunchLog lg;
    explicit CallLog(afc_ctx* c) : ctx(c) {
        if (ctx->profile) { lg.profile = true; lg.pool = ctx->prof_recs.data(); lg.cap = (int)ctx->prof_recs.size(); lg.next = &ctx->prof_next; }
    }
    ~CallLog() { ctx->launches += lg.n; }
    operator launch::LaunchLog*() { return &lg; }
};


// ---- issuer-key cache management ------------------------------------------------------------------------------
void kc_free_call_buffers(launch::KeyCache& k) {
    void* ps[] = {k.bslots, k.rep, k.kid, k.cnt, k.dlist, k.cand, k.perm, k.cold, k.pts};
    for (void* p : ps) if (p) cudaFree(p);
    k.bslots = k.rep = k.kid = k.cnt = k.dlist = k.cand = k.perm = k.cold = nullptr; k.pts = nullptr;
}
void kc_free(afc_ctx* ctx) {
    launch::KeyCache& k = ctx->kc;
    void* ps[] = {k.slots, k.cpks, k.valid, k.tabs, k.stamp, k.free_list, k.bucket, k.state, k.build_list, k.bases};
    for (void* p : ps) if (p) cudaFree(p);
    kc_free_call_buffers(k);
    if (k.side) cudaStreamDestroy(k.side);
    if (k.side2) cudaStreamDestroy(k.side2);
    cudaEvent_t evs[] = {k.ev_fork, k.ev_join, k.ev_plan, k.ev_rows, k.ev_chain[0], k.ev_chain[1], k.ev_chain[2], k.ev_chain[3]};
    for (cudaEvent_t e : evs) if (e) cudaEventDestroy(e);
    k = launch::KeyCache{};
    ctx->kc_ready = false; ctx->kc_call_cap = 0;
}
// Makes the cache usable for a call of n items (allocating / growing as needed).  Returns nullptr when disabled or when
// memory cannot be had — callers then run the generic kernel.  Caller holds kc_mu.
const launch::KeyCache* kc_prepare(afc_ctx* ctx, uint32_t n) {
    if (ctx->kc_max_keys == 0 || n < 64) return nullptr;
    launch::KeyCache& k = ctx->kc;
    auto dmalloc = [](auto** p, size_t bytes) { return cudaMalloc((void**)p, bytes ? bytes : 1) == cudaSuccess; };
    if (!ctx->kc_ready) {
        uint32_t cap = 1; while (cap < 4 * (uint64_t)ctx->kc_max_keys) cap <<= 1;
        k.slot_mask = cap - 1; k.max_keys = ctx->kc_max_keys;
        const size_t mk = k.max_keys;
        int prio_least = 0, prio_greatest = 0;
        bool ok = dmalloc(&k.slots, (size_t)cap * 4) && dmalloc(&k.cpks, mk * 32) && dmalloc(&k.valid, mk) &&
                  dmalloc(&k.tabs, launch::ed_key_table_bytes(k.max_keys)) && dmalloc(&k.stamp, mk * 4) && dmalloc(&k.free_list, mk * 4) &&
                  dmalloc(&k.bucket, (mk + 1) * 4) && dmalloc(&k.state, launch::KS_WORDS * 4) && dmalloc(&k.build_list, mk * 4) &&
                  dmalloc(&k.bases, launch::ed_key_bases_bytes(k.max_keys)) &&
                  cudaMemset(k.slots, 0xff, (size_t)cap * 4) == cudaSuccess && cudaMemset(k.state, 0, launch::KS_WORDS * 4) == cudaSuccess &&
                  cudaMemset(k.valid, 0, mk) == cudaSuccess && cudaMemset(k.stamp, 0, mk * 4) == cudaSuccess &&
                  cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest) == cudaSuccess &&
                  cudaStreamCreateWithPriority(&k.side, cudaStreamNonBlocking, prio_greatest) == cudaSuccess &&
                  cudaStreamCreateWithPriority(&k.side2, cudaStreamNonBlocking, prio_greatest) == cudaSuccess &&
                  (ctx->kc_event || cudaEventCreateWithFlags(&ctx->kc_event, cudaEventDisableTiming) == cudaSuccess);
        cudaEvent_t* evs[] = {&k.ev_fork, &k.ev_join, &k.ev_plan, &k.ev_rows, &k.ev_chain[0], &k.ev_chain[1], &k.ev_chain[2], &k.ev_chain[3]};
        for (cudaEvent_t* e : evs) ok = ok && cudaEventCreateWithFlags(e, cudaEventDisableTiming) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(cudaStreamLegacy) == cudaSuccess;        // the memsets above vs the non-blocking side streams
        if (!ok) { cudaGetLastError(); kc_free(ctx); ctx->kc_max_keys = 0; return nullptr; }     // no room: stay generic
        ctx->kc_ready = true;
    }
    if (n > ctx->kc_call_cap) {
        // earlier calls may still be using the per-call buffers on their streams: wait for the last cache user before freeing
        if (ctx->kc_call_cap) { cudaEventSynchronize(ctx->kc_event); }
        kc_free_call_buffers(k);
        const uint64_t want = (uint64_t)n + n / 4;
        uint64_t cap = 1; while (cap < 2 * want) cap <<= 1;
        if (cap > 0x80000000ull) { ctx->kc_call_cap = 0; return nullptr; }                    // beyond the 32-bit tables: generic kernel
        bool ok = dmalloc(&k.bslots, (size_t)cap * 4) && dmalloc(&k.rep, want * 4) && dmalloc(&k.kid, want * 4) && dmalloc(&k.cnt, want * 4) &&
                  dmalloc(&k.dlist, want * 4) && dmalloc(&k.cand, want * 4) && dmalloc(&k.perm, want * 4) && dmalloc(&k.cold, want * 4) &&
                  (launch::ed_verify_pts_bytes(want) == 0 || dmalloc(&k.pts, launch::ed_verify_pts_bytes(want)));
        if (!ok) { cudaGetLastError(); kc_free_call_buffers(k); ctx->kc_call_cap = 0; return nullptr; }
        k.bmask = (uint32_t)(cap - 1); ctx->kc_call_cap = (uint32_t)(want > 0xffffffffull ? 0xffffffffu : want);
    }
    return &k;
}
// verify through the cache when possible; serialises cache users across streams with an event
cudaError_t verify_with_cache(afc_ctx* ctx, const uint8_t* pks, const uint8_t* sigs, const uint8_t* msgs, const uint64_t* off, uint32_t n,
                              uint8_t* ok, uint32_t* scratch_k, cudaStream_t st, launch::LaunchLog* lg) {
    std::lock_guard<std::mutex> g(ctx->kc_mu);
    const launch::KeyCache* kc = kc_prepare(ctx, n);
    if (kc) { cudaError_t e = cudaStreamWaitEvent(st, ctx->kc_event, 0); if (e != cudaSuccess) return e; }
    cudaError_t e = launch::ed_verify_batch(ctx->comb, pks, sigs, msgs, off, n, ok, scratch_k, kc, st, lg);
    if (kc && e == cudaSuccess) e = cudaEventRecord(ctx->kc_event, st);
    return e;
}

struct LaneGuard {
    afc_ctx* ctx; int idx;
    LaneGuard(afc_ctx* c) : ctx(c), idx(-1) {
        std::unique_lock<std::mutex> lk(ctx->mu);
        for (;;) {
            for (int i = 0; i < kLanes; i++) if (!ctx->lanes[i].busy) { idx = i; break; }
            if (idx >= 0) break;
            ctx->cv.wait(lk);
        }
        ctx->lanes[idx].busy = true;
    }
    ~LaneGuard() {
        { std::lock_guard<std::mutex> g(ctx->mu); ctx->lanes[idx].busy = false; }
        ctx->cv.notify_one();
    }
    Lane& lane() { return ctx->lanes[idx]; }
};

bool is_pinned(const void* p) {
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return at.type == cudaMemoryTypeHost;
}

inline bool aligned16(const void* p) { return (((uintptr_t)p) & 15) == 0; }

#define RC(expr)                                                           \
    do {                                                                   \
        const int _rc = (expr);                                            \
        if (_rc != AFC_OK) return _rc;                                     \
    } while (0)

// ---- per-call scratch layouts
size_t vc_align(size_t x) { return (x + 255) & ~(size_t)255; }
typedef std::vector<std::pair<uint8_t*, size_t>> Regions;
// A layout is written once and run twice: over a Carve without a base it only adds up the 256-aligned sizes (what to reserve), over one
// with a base it hands out the pointers in the same order.  Regions taken as secret join `secrets` when the carver keeps that list.
struct Carve {
    uint8_t* base = nullptr;
    size_t used = 0;
    Regions* secrets = nullptr;
    uint8_t* take(size_t bytes, bool secret = false) {
        uint8_t* p = base ? base + used : nullptr;
        if (p && secret && secrets) secrets->push_back({p, vc_align(bytes)});
        used += vc_align(bytes);
        return p;
    }
    template <class T> T* take(size_t count, bool secret = false) { return (T*)take(count * sizeof(T), secret); }
};
// A _dev call's scratch: sized by the layout, allocated from the stream-ordered pool, carved by the same layout (the caller frees it)
template <class Layout> cudaError_t pool_carve(uint8_t** scratch, cudaStream_t st, Layout&& layout) {
    Carve m;
    layout(m);
    const cudaError_t e = cudaMallocAsync((void**)scratch, m.used, st);
    if (e != cudaSuccess) return e;
    Carve k;
    k.base = *scratch;
    layout(k);
    return cudaSuccess;
}

// ---- stored credential documents: parse -> scan -> emit -> keyed verify -> fold, in one scratch area
// The signing messages of a batch are never longer than its documents (D[0:p] plus the zero-proof text, which is no longer than the proof
// object it replaces), so doc_bytes bounds their buffer.  k_vcj_parse / k_vcj_emit decline a message longer than its document, so the same
// bound holds for documents in any spelling.  The audit (`audit`) also captures each document for k_vc_crosscheck.
struct VcScratch { uint8_t* msgs; uint64_t* msg_off; uint8_t* sigs; uint32_t* kidx; uint8_t* ok; uint64_t* scan; uint32_t* kscr; uint32_t* caps; };
void vc_scratch(Carve& k, VcScratch& s, uint32_t n, uint64_t doc_bytes, uint32_t n_keys, bool audit) {
    s.msgs = k.take(doc_bytes + 64);
    s.msg_off = k.take<uint64_t>((size_t)n + 1);
    s.sigs = k.take((size_t)n * 64);
    s.kidx = k.take<uint32_t>(n);
    s.ok = k.take(n);
    s.scan = (uint64_t*)k.take(launch::json_scan_scratch_bytes(n));
    s.kscr = (uint32_t*)k.take((size_t)n * 32 + launch::ed_keyed_scratch_bytes(n_keys, n));
    s.caps = audit ? (uint32_t*)k.take(launch::vc_capture_bytes(n)) : nullptr;
}
// docs + doc_off[i] is document i (absolute offsets).  With `issues` (the audit) the parse also captures each document and k_vc_crosscheck
// compares it with its record's columns; the scratch is then carved with `audit`.  With `json` (afc_vc_verify_json_batch) documents in any
// spelling are read and re-marshalled by k_vcj_parse / k_vcj_emit.
cudaError_t vc_stored_enqueue(afc_ctx* ctx, const afc_keyset* ks, int kind, const uint8_t* docs, const uint64_t* doc_off, uint32_t n,
                              uint8_t* status, uint32_t* fields, const VcScratch& S, cudaStream_t st, launch::LaunchLog* lg,
                              uint32_t* issues = nullptr, const uint8_t* cols = nullptr, const uint64_t* col_off = nullptr, bool json = false) {
    if (n == 0) return cudaSuccess;
    const void* schema = ks->d_schemas + (size_t)kind * launch::vc_schema_bytes();
    const void* jschema = ks->d_vcj_schemas + (size_t)kind * launch::vcj_schema_bytes();
    cudaError_t e;
    if (json) {
        e = launch::vcj_parse(jschema, docs, doc_off, n, ks->d_dids, ks->d_did_off, ks->d_slots, ks->slot_mask, status, S.msg_off + 1, S.sigs,
                              S.kidx, fields, st, lg);
    } else if (issues) {
        e = launch::vc_parse_capture(schema, docs, doc_off, n, ks->d_dids, ks->d_did_off, ks->d_slots, ks->slot_mask, status, S.msg_off + 1, S.sigs,
                                     S.kidx, S.caps, st, lg);
        if (e == cudaSuccess) e = launch::vc_crosscheck(kind, docs, doc_off, n, S.caps, status, cols, col_off, issues, st, lg);
    } else {
        e = launch::vc_parse(schema, docs, doc_off, n, ks->d_dids, ks->d_did_off, ks->d_slots, ks->slot_mask, status, S.msg_off + 1, S.sigs,
                             S.kidx, fields, st, lg);
    }
    if (e == cudaSuccess) e = launch::offsets_from_lengths(S.msg_off, n, S.scan, st, lg);
    if (e == cudaSuccess) e = json ? launch::vcj_emit(jschema, docs, doc_off, n, S.msg_off, S.msgs, st, lg)
                                   : launch::vc_emit(schema, docs, doc_off, n, S.msg_off, S.msgs, st, lg);
    if (e == cudaSuccess) e = launch::ed_verify_keyed_batch(ctx->comb, ks->d_tabs, ks->d_valid, ks->d_pks, ks->n_keys, S.kidx, S.sigs, S.msgs,
                                                            S.msg_off, n, S.ok, S.kscr, S.kscr + (size_t)n * 8, st, lg);
    if (e == cudaSuccess) e = launch::vc_fold(status, S.ok, n, st, lg);
    return e;
}

// offsets must be non-decreasing: a caller's slip would otherwise turn into an out-of-bounds copy from its own buffer
template <class T>
bool monotone(const T* off, uint32_t n) {
    T bad = 0;
    for (uint32_t i = 0; i < n; i++) bad |= (T)(off[i + 1] < off[i]);
    return bad == 0;
}

// AFC_CHUNK_ITEMS / AFC_MIN_CHUNK_ITEMS: tuning knobs for experiments (read once per process)
uint32_t max_chunk_items() {
    static const uint32_t v = [] { const char* e = getenv("AFC_CHUNK_ITEMS"); uint32_t x = e ? (uint32_t)strtoul(e, nullptr, 10) : 0; return x ? x : kChunkItems; }();
    return v;
}
uint32_t min_chunk_items() {
    static const uint32_t v = [] { const char* e = getenv("AFC_MIN_CHUNK_ITEMS"); uint32_t x = e ? (uint32_t)strtoul(e, nullptr, 10) : 0; return x ? x : kMinChunkItems; }();
    return v;
}

constexpr uint64_t kBadOffsets = ~0ull;     // a chunk measure's answer when an item's offsets run backwards

// An output of a chunk: `bytes` from device `src` to `arg` + `at` in the caller's memory; with `offsets`, uint64 offsets rebased by `base`
struct Out {
    void* arg; size_t at; const void* src; size_t bytes;
    bool secret = false;
    bool offsets = false; uint64_t base = 0;
};
Out offsets_out(uint64_t* arg, size_t first, const uint64_t* src, size_t count, uint64_t base) {
    return {arg, first * 8, src, count * 8, false, true, base};
}

// The staging pipeline of every host-buffer call.  It holds a lane and runs the call's chunks through `depth` of its slots, so that the
// copies of later chunks overlap the kernels of earlier ones.  A chunk's function stages its inputs and carves its scratch (stage),
// enqueues its kernels on `st`, and names its outputs (copy_back); the ring moves the bytes, through the slot's bounce buffers when the
// caller's memory is pageable, and wipes whatever was marked secret:
// - its device bytes on the slot's stream once the chunk's copy-back is enqueued;
// - its bounce bytes once the slot has been synchronised;
// - both, after every stream of the lane has drained, on any early return.
// On ANY exit, error paths included, nothing may still be reading the caller's buffers or writing its results: every stream the call used
// is drained before the lane is handed to the next caller.
class Ring {
public:
    // Carves a chunk's slot arena and stages its inputs: a layout runs twice, measuring then carving (Carve)
    struct Stager : Carve {
        Ring* r = nullptr;
        size_t bounce = 0;                  // bytes of the input bounce buffer: measured, then filled
        cudaError_t err = cudaSuccess;
        // arg[first, first + count): the result is the staged copy of arg[first]
        template <class T> T* in(const T* arg, size_t first, size_t count, bool secret = false) {
            return (T*)r->stage_in(*this, arg, first * sizeof(T), count * sizeof(T), count * sizeof(T) + 16, 0, secret);
        }
        // arg[first, first + bytes), congruent mod `mod` (16, or 4 for keys) with its absolute offsets: the result + first is the first byte,
        // so that absolute offsets stay valid and the kernels see the alignment of the caller's buffer whatever the chunking
        uint8_t* in_at(const uint8_t* arg, uint64_t first, uint64_t bytes, unsigned mod, bool secret = false) {
            uint8_t* p = r->stage_in(*this, arg, first, bytes, bytes + 32, first & (mod - 1), secret);
            return p ? p - first : nullptr;
        }
    };

    afc_ctx* const ctx;
    CallLog lc;
    uint32_t i0 = 0, cnt = 0;               // the chunk being run: items [i0, i0 + cnt)
    cudaStream_t st = nullptr;

    explicit Ring(afc_ctx* c, int depth = kSlots) : ctx(c), lc(c), lane_(c), depth_(depth) {}
    ~Ring() {
        if (!armed_) return;
        Lane& lane = lane_.lane();
        for (int w = 0; w < depth_; w++) cudaStreamSynchronize(lane.slot[w].stream);
        for (int w = 0; w < depth_; w++) {
            for (const auto& s : pend_[w].dev_secrets) cudaMemsetAsync(s.first, 0, s.second, lane.slot[w].stream);
            cudaStreamSynchronize(lane.slot[w].stream);
            for (const auto& s : pend_[w].host_secrets) memset(s.first, 0, s.second);
        }
    }

    // The chunk walk: each chunk takes at most max_chunk_items() items and, with more than one slot, at most half of what is left, down to
    // min_chunk_items() (what remains after the last H2D copy lands, the part of a transfer-bound call that nothing overlaps, stays small);
    // and no more items than keep measure(i0, i) — the bytes of items [i0, i] — within kChunkBytes, but always at least one.  The walk that
    // sizes a chunk is also where its offsets are checked (measure returns kBadOffsets), so no separate pass reads them.
    template <class Measure, class Fn> int walk(uint32_t n, Measure&& measure, Fn&& fn) {
        const uint32_t max_chunk = max_chunk_items(), min_chunk = min_chunk_items();
        for (uint32_t a = 0, b; a < n; a = b) {
            const uint32_t left = n - a;
            uint32_t limit = max_chunk;
            if (depth_ > 1) {
                limit = left <= min_chunk ? left : (left + 1) / 2;
                if (limit < min_chunk) limit = min_chunk;
                if (limit > max_chunk) limit = max_chunk;
            }
            for (b = a; b < n && b - a < limit; b++) {
                const uint64_t bytes = measure(a, b);
                if (bytes == kBadOffsets) return AFC_EINVAL;
                if (bytes > kChunkBytes && b != a) break;
            }
            RC(chunk(a, b - a, fn));
        }
        return finish();
    }
    // all n items as one chunk
    template <class Fn> int once(uint32_t n, Fn&& fn) {
        RC(chunk(0, n, fn));
        return finish();
    }

    template <class Layout> int stage(Layout&& layout) {
        Stager m;
        m.r = this;
        layout(m);
        Slot& sl = slot();
        CK(sl.arena.reserve(m.used));
        CK(sl.h_in.reserve(m.bounce + 256, ctx));
        Stager k;
        k.r = this; k.base = sl.arena.p; k.secrets = &pend_[which_].dev_secrets;
        layout(k);
        CK(k.err);
        return AFC_OK;
    }
    // reads the values at src into dst (where the chunk's outputs end): synchronises the slot's stream
    int read(uint64_t* dst, std::initializer_list<const uint64_t*> src) {
        Slot& sl = slot();
        CK(sl.h_out.reserve(src.size() * 8, ctx));
        size_t k = 0;
        for (const uint64_t* s : src) CK(cudaMemcpyAsync(sl.h_out.p + 8 * k++, s, 8, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        memcpy(dst, sl.h_out.p, src.size() * 8);
        return AFC_OK;
    }
    // enqueues the chunk's outputs; what goes through the output bounce reaches the caller when the slot is drained
    int copy_back(std::initializer_list<Out> outs) {
        Slot& sl = slot();
        Pending& p = pend_[which_];
        size_t bounce = 0;
        for (const Out& o : outs) if (o.bytes && (o.offsets || !pinned(o.arg))) bounce += vc_align(o.bytes);
        CK(sl.h_out.reserve(bounce + 256, ctx));
        uint8_t* h = sl.h_out.p;
        for (const Out& o : outs) {
            if (!o.bytes) continue;
            uint8_t* dst = (uint8_t*)o.arg + o.at;
            if (o.offsets || !pinned(o.arg)) {
                p.back.push_back({dst, h, o.bytes, o.offsets, o.base});
                if (o.secret) p.host_secrets.push_back({h, o.bytes});
                dst = h;
                h += vc_align(o.bytes);
            }
            CK(cudaMemcpyAsync(dst, o.src, o.bytes, cudaMemcpyDeviceToHost, st));
        }
        return AFC_OK;
    }

private:
    struct Back { uint8_t* dst; const uint8_t* src; size_t bytes; bool offsets; uint64_t base; };
    struct Pending {
        bool active = false;
        std::vector<Back> back;             // outputs waiting in the output bounce
        Regions dev_secrets, host_secrets;
    };
    LaneGuard lane_;
    const int depth_;
    int which_ = 0;
    bool armed_ = true;
    Pending pend_[kSlots];
    std::vector<std::pair<const void*, bool>> pinned_;      // each argument's memory type, looked up once per call

    Slot& slot() { return lane_.lane().slot[which_]; }
    bool pinned(const void* arg) {
        for (const auto& a : pinned_) if (a.first == arg) return a.second;
        pinned_.push_back({arg, is_pinned(arg)});
        return pinned_.back().second;
    }
    uint8_t* stage_in(Stager& k, const void* arg, size_t at, size_t bytes, size_t region, size_t pad, bool secret) {
        uint8_t* d = k.take(region, secret);
        const bool direct = bytes == 0 || pinned(arg);
        if (!k.base) {
            if (!direct) k.bounce += vc_align(bytes);
            return nullptr;
        }
        if (bytes == 0 || k.err != cudaSuccess) return d + pad;
        const uint8_t* src = (const uint8_t*)arg + at;
        if (!direct) {
            uint8_t* h = slot().h_in.p + k.bounce;
            memcpy(h, src, bytes);
            if (secret) pend_[which_].host_secrets.push_back({h, bytes});
            k.bounce += vc_align(bytes);
            src = h;
        }
        k.err = cudaMemcpyAsync(d + pad, src, bytes, cudaMemcpyHostToDevice, st);
        return d + pad;
    }
    template <class Fn> int chunk(uint32_t a, uint32_t n, Fn&& fn) {
        RC(drain(which_));
        i0 = a; cnt = n; st = slot().stream;
        Pending& p = pend_[which_];
        p.active = true;
        RC(fn(*this));
        for (const auto& s : p.dev_secrets) CK(cudaMemsetAsync(s.first, 0, s.second, st));
        which_ = (which_ + 1) % depth_;
        return AFC_OK;
    }
    int drain(int w) {
        Pending& p = pend_[w];
        if (!p.active) return AFC_OK;
        CK(cudaStreamSynchronize(lane_.lane().slot[w].stream));
        for (const Back& b : p.back) {
            if (!b.offsets) { memcpy(b.dst, b.src, b.bytes); continue; }
            for (size_t j = 0; j < b.bytes / 8; j++) ((uint64_t*)b.dst)[j] = b.base + ((const uint64_t*)b.src)[j];
        }
        for (const auto& s : p.host_secrets) memset(s.first, 0, s.second);
        p.active = false;
        p.back.clear(); p.dev_secrets.clear(); p.host_secrets.clear();
        return AFC_OK;
    }
    int finish() {
        for (int w = 0; w < depth_; w++) RC(drain((which_ + w) % depth_));      // oldest first
        armed_ = false;
        return AFC_OK;
    }
};
typedef Ring::Stager Stager;

// A chunk of messages and their offsets (msgs + off[i] is message i, absolute offsets), and the walk's measure over them
struct Msgs { const uint8_t* d; const uint64_t* off; };
Msgs stage_msgs(Stager& k, const uint8_t* msgs, const uint64_t* off, uint32_t i0, uint32_t cnt) {
    return {k.in_at(msgs, off[i0], off[i0 + cnt] - off[i0], 16), k.in(off, i0, (size_t)cnt + 1)};
}
auto msg_bytes(const uint64_t* off) {
    return [off](uint32_t i0, uint32_t i) { return off[i + 1] < off[i] ? kBadOffsets : off[i + 1] - off[i0]; };
}

// Expanded private keys for a host-buffer call: on the device once for every chunk, zeroed and freed when the call returns
template <class Fn> int with_device_keys(afc_ctx* ctx, const uint8_t* expanded96, uint32_t n_keys, Fn&& run) {
    uint8_t* d_keys = nullptr;
    CK(cudaMalloc(&d_keys, (size_t)n_keys * 96));
    const cudaError_t e = cudaMemcpy(d_keys, expanded96, (size_t)n_keys * 96, cudaMemcpyHostToDevice);
    int rc = AFC_ECUDA;
    if (e == cudaSuccess) rc = run(d_keys);
    else set_err(ctx, e, "cudaMemcpy(expanded keys)");
    cudaMemset(d_keys, 0, (size_t)n_keys * 96);
    cudaFree(d_keys);
    return rc;
}

}  // namespace

// Binds the CALLING THREAD to the CPUs next to ctx's GPU for the lifetime of the scope: pages allocated (and pinned) meanwhile
// land on that GPU's NUMA node.  One process driving 8 contexts (the Go control plane) otherwise stages half of its batches
// through the far socket, at a fraction of the local copy rate.
struct NumaScope {
    cpu_set_t old; bool active = false;
    explicit NumaScope(afc_ctx* ctx) {
        static const bool off = [] { const char* e = getenv("AFC_NUMA_BIND"); return e && atoi(e) == 0; }();
        if (!ctx || !ctx->has_local_cpus || off) return;
        if (sched_getaffinity(0, sizeof old, &old) != 0) return;
        cpu_set_t want; CPU_AND(&want, &old, &ctx->local_cpus);
        if (CPU_COUNT(&want) == 0 || CPU_EQUAL(&want, &old)) return;
        active = sched_setaffinity(0, sizeof want, &want) == 0;
    }
    ~NumaScope() { if (active) sched_setaffinity(0, sizeof old, &old); }
};
void* afc_internal_pinned_alloc(afc_ctx* ctx, size_t bytes) {
    NumaScope ns(ctx);
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
static void numa_discover(afc_ctx* ctx) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, ctx->device) != cudaSuccess) { cudaGetLastError(); return; }
    for (char* c = bus; *c; c++) if (*c >= 'A' && *c <= 'F') *c = (char)(*c - 'A' + 'a');
    std::string base = std::string("/sys/bus/pci/devices/") + bus;
    if (FILE* f = fopen((base + "/numa_node").c_str(), "r")) { if (fscanf(f, "%d", &ctx->numa_node) != 1) ctx->numa_node = -1; fclose(f); }
    FILE* f = fopen((base + "/local_cpulist").c_str(), "r");
    if (!f) return;
    char line[4096] = {0};
    if (fgets(line, sizeof line, f)) {
        CPU_ZERO(&ctx->local_cpus);
        int n = 0;
        for (char* tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
            int a = 0, b = 0;
            if (sscanf(tok, "%d-%d", &a, &b) == 2) { for (int c = a; c <= b && c < CPU_SETSIZE; c++) { CPU_SET(c, &ctx->local_cpus); n++; } }
            else if (sscanf(tok, "%d", &a) == 1 && a < CPU_SETSIZE) { CPU_SET(a, &ctx->local_cpus); n++; }
        }
        ctx->has_local_cpus = n > 0;
    }
    fclose(f);
}

int afc_internal_device(afc_ctx* ctx) { return ctx->device; }
const void* afc_internal_comb(afc_ctx* ctx) { return ctx->comb; }
const void* afc_internal_sign_table(afc_ctx* ctx) { return ctx->sign_ct ? ctx->ct16 : nullptr; }
void afc_internal_add_launches(afc_ctx* ctx, unsigned long long n) { ctx->launches += n; }

extern "C" {

const char* afc_version(void) { return "afcrypto-b200 0.1.0 (sm_90a)"; }

const char* afc_strerror(int rc) {
    switch (rc) {
    case AFC_OK: return "ok";
    case AFC_EINVAL: return "invalid argument";
    case AFC_ECUDA: return "CUDA failure (see afc_last_cuda_error)";
    case AFC_ENOMEM: return "out of memory";
    case AFC_ENCCL: return "NCCL failure or NCCL unavailable";
    case AFC_ESTATE: return "invalid state";
    default: return "unknown error";
    }
}

const char* afc_last_cuda_error(afc_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "no context"; }

int afc_init(int device, afc_ctx** out) {
    if (!out) return AFC_EINVAL;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return AFC_ECUDA; }
    if (device < 0 || device >= ndev) return AFC_EINVAL;
    afc_ctx* ctx = new (std::nothrow) afc_ctx();
    if (!ctx) return AFC_ENOMEM;
    ctx->device = device;
    if (const char* e = getenv("AFC_KEYCACHE_MAX_KEYS")) ctx->kc_max_keys = (uint32_t)strtoul(e, nullptr, 10);
    auto fail = [&](cudaError_t e, const char* what) { set_err(ctx, e, what); fprintf(stderr, "afc_init: %s\n", ctx->last_error.c_str()); afc_destroy(ctx); return AFC_ECUDA; };
    cudaError_t e;
    if ((e = cudaSetDevice(device)) != cudaSuccess) return fail(e, "cudaSetDevice");
    if ((e = cudaGetDeviceProperties(&ctx->prop, device)) != cudaSuccess) return fail(e, "cudaGetDeviceProperties");
    numa_discover(ctx);
    {   // per-call scratch comes from the stream-ordered pool: keep freed blocks across synchronisations instead of returning them to
        // the driver (the default threshold of 0 re-maps the 32 MB of a 1 M-credential call after every sync)
        cudaMemPool_t pool = nullptr;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess && pool) {
            unsigned long long keep = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        cudaGetLastError();
    }
    for (int l = 0; l < kLanes; l++)
        for (int s = 0; s < kSlots; s++)
            if ((e = cudaStreamCreateWithFlags(&ctx->lanes[l].slot[s].stream, cudaStreamNonBlocking)) != cudaSuccess) return fail(e, "cudaStreamCreate");
    if ((e = cudaMalloc(&ctx->comb, launch::ed_tables_bytes())) != cudaSuccess) return fail(e, "cudaMalloc(tables)");
    cudaStream_t s0 = ctx->lanes[0].slot[0].stream;
    if ((e = cudaMalloc(&ctx->ct16, launch::ed_ct_table_bytes())) != cudaSuccess) return fail(e, "cudaMalloc(ct table)");
    if (const char* ev = getenv("AFC_SIGN_CT")) ctx->sign_ct = atoi(ev) != 0;
    {   // the launch log must be gone before fail() can destroy the context it points into
        CallLog lc(ctx);
        e = launch::ed_build_tables(ctx->comb, s0, lc);
        if (e == cudaSuccess) e = launch::ed_build_ct_table(ctx->comb, ctx->ct16, s0, lc);
    }
    if (e != cudaSuccess) return fail(e, "ed_build_tables");
    if ((e = cudaStreamSynchronize(s0)) != cudaSuccess) return fail(e, "ed_build_tables sync");
    *out = ctx;
    return AFC_OK;
}

void afc_destroy(afc_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    afc_comm_destroy(ctx);
    for (int l = 0; l < kLanes; l++)
        for (int s = 0; s < kSlots; s++) {
            Slot& sl = ctx->lanes[l].slot[s];
            if (sl.stream) { cudaStreamSynchronize(sl.stream); cudaStreamDestroy(sl.stream); }
            sl.arena.release(); sl.h_in.release(); sl.h_out.release();
        }
    kc_free(ctx);
    if (ctx->kc_event) cudaEventDestroy(ctx->kc_event);
    if (ctx->comb) cudaFree(ctx->comb);
    if (ctx->ct16) cudaFree(ctx->ct16);
    for (auto& r : ctx->prof_recs) { if (r.e0) cudaEventDestroy(r.e0); if (r.e1) cudaEventDestroy(r.e1); }
    delete ctx;
}

int afc_device_info(afc_ctx* ctx, int* sm_count, int* clock_khz, uint64_t* mem_bytes) {
    if (!ctx) return AFC_EINVAL;
    if (sm_count) *sm_count = ctx->prop.multiProcessorCount;
    if (clock_khz) { int v = 0; cudaDeviceGetAttribute(&v, cudaDevAttrClockRate, ctx->device); *clock_khz = v; }
    if (mem_bytes) *mem_bytes = ctx->prop.totalGlobalMem;
    return AFC_OK;
}

int afc_sign_configure(afc_ctx* ctx, int constant_time) {
    if (!ctx) return AFC_EINVAL;
    ctx->sign_ct = constant_time != 0;
    return AFC_OK;
}
int afc_sign_mode(afc_ctx* ctx) { return ctx ? (ctx->sign_ct ? 1 : 0) : AFC_EINVAL; }

uint64_t afc_launch_count(afc_ctx* ctx) { return ctx ? (uint64_t)ctx->launches.load() : 0; }

void* afc_alloc_pinned(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void afc_free_pinned(void* p) { if (p) cudaFreeHost(p); }
void* afc_alloc_pinned_for(afc_ctx* ctx, size_t bytes) { return ctx ? afc_internal_pinned_alloc(ctx, bytes) : nullptr; }
int afc_numa_info(afc_ctx* ctx, int* numa_node, int* local_cpus) {
    if (!ctx) return AFC_EINVAL;
    if (numa_node) *numa_node = ctx->numa_node;
    if (local_cpus) *local_cpus = ctx->has_local_cpus ? CPU_COUNT(&ctx->local_cpus) : 0;
    return AFC_OK;
}

// ---------------------------------------------------------------------------------- host-buffer batch calls
int afc_sha256_batch(afc_ctx* ctx, const uint8_t* msgs, const uint64_t* offsets, uint32_t n, uint8_t* out32) {
    if (!ctx || !offsets || (!out32 && n) || (!msgs && n && offsets[n] != offsets[0])) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    CK(cudaSetDevice(ctx->device));
    Ring ring(ctx);
    return ring.walk(n, msg_bytes(offsets), [&](Ring& r) {
        Msgs M;
        uint8_t* d_out;
        RC(r.stage([&](Stager& k) {
            M = stage_msgs(k, msgs, offsets, r.i0, r.cnt);
            d_out = k.take((size_t)r.cnt * 32 + 16);
        }));
        CK(launch::sha256_batch(M.d, M.off, r.cnt, d_out, r.st, r.lc));
        return r.copy_back({{out32, (size_t)r.i0 * 32, d_out, (size_t)r.cnt * 32}});
    });
}
int afc_hmac_sha256_batch(afc_ctx* ctx, const uint8_t* keys, const uint32_t* key_off, const uint8_t* msgs,
                          const uint64_t* msg_off, uint32_t n, uint8_t* out32) {
    if (!ctx || !key_off || !msg_off || (!out32 && n)) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    if (!monotone(key_off, n)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    Ring ring(ctx);
    return ring.walk(n, msg_bytes(msg_off), [&](Ring& r) {
        Msgs M;
        const uint8_t* d_keys;
        const uint32_t* d_koff;
        uint8_t* d_out;
        RC(r.stage([&](Stager& k) {
            M = stage_msgs(k, msgs, msg_off, r.i0, r.cnt);
            d_keys = k.in_at(keys, key_off[r.i0], key_off[r.i0 + r.cnt] - key_off[r.i0], 4);
            d_koff = k.in(key_off, r.i0, (size_t)r.cnt + 1);
            d_out = k.take((size_t)r.cnt * 32 + 16);
        }));
        CK(launch::hmac_sha256_batch(d_keys, d_koff, M.d, M.off, r.cnt, d_out, r.st, r.lc));
        return r.copy_back({{out32, (size_t)r.i0 * 32, d_out, (size_t)r.cnt * 32}});
    });
}
int afc_ed25519_verify_batch(afc_ctx* ctx, const uint8_t* pks, const uint8_t* sigs, const uint8_t* msgs,
                             const uint64_t* msg_off, uint32_t n, uint8_t* ok) {
    if (!ctx || !msg_off || (n && (!pks || !sigs || !ok))) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    CK(cudaSetDevice(ctx->device));
    Ring ring(ctx);
    return ring.walk(n, msg_bytes(msg_off), [&](Ring& r) {
        Msgs M;
        const uint8_t *d_pks, *d_sigs;
        uint8_t* d_ok;
        uint32_t* d_k;
        RC(r.stage([&](Stager& k) {
            M = stage_msgs(k, msgs, msg_off, r.i0, r.cnt);
            d_pks = k.in(pks, (size_t)r.i0 * 32, (size_t)r.cnt * 32);
            d_sigs = k.in(sigs, (size_t)r.i0 * 64, (size_t)r.cnt * 64);
            d_ok = k.take((size_t)r.cnt + 16);
            d_k = k.take<uint32_t>((size_t)r.cnt * 8);
        }));
        CK(verify_with_cache(ctx, d_pks, d_sigs, M.d, M.off, r.cnt, d_ok, d_k, r.st, r.lc));
        return r.copy_back({{ok, r.i0, d_ok, r.cnt}});
    });
}
int afc_ed25519_sign_batch(afc_ctx* ctx, const uint8_t* seeds, const uint8_t* msgs, const uint64_t* msg_off,
                           uint32_t n, uint8_t* sigs) {
    if (!ctx || !msg_off || (n && (!seeds || !sigs))) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    CK(cudaSetDevice(ctx->device));
    Ring ring(ctx);
    return ring.walk(n, msg_bytes(msg_off), [&](Ring& r) {
        Msgs M;
        const uint8_t* d_seeds;
        uint8_t* d_sigs;
        RC(r.stage([&](Stager& k) {
            M = stage_msgs(k, msgs, msg_off, r.i0, r.cnt);
            d_seeds = k.in(seeds, (size_t)r.i0 * 32, (size_t)r.cnt * 32, true);
            d_sigs = k.take((size_t)r.cnt * 64 + 16);
        }));
        CK(launch::ed_sign_batch(ctx->comb, afc_internal_sign_table(ctx), d_seeds, M.d, M.off, r.cnt, d_sigs, r.st, r.lc));
        return r.copy_back({{sigs, (size_t)r.i0 * 64, d_sigs, (size_t)r.cnt * 64}});
    });
}

// ---------------------------------------------------------------------------------- H2: streaming SHA-256
int afc_sha256_stream_init(uint8_t* states, uint32_t n) {
    if (!states && n) return AFC_EINVAL;
    static const uint32_t iv[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    for (uint32_t i = 0; i < n; i++) {
        uint8_t* s = states + (size_t)AFC_SHA256_STATE_BYTES * i;
        memset(s, 0, AFC_SHA256_STATE_BYTES);
        s[0] = 's'; s[1] = 'h'; s[2] = 'a'; s[3] = 3;
        for (int w = 0; w < 8; w++) { s[4 + 4 * w] = (uint8_t)(iv[w] >> 24); s[5 + 4 * w] = (uint8_t)(iv[w] >> 16); s[6 + 4 * w] = (uint8_t)(iv[w] >> 8); s[7 + 4 * w] = (uint8_t)iv[w]; }
    }
    return AFC_OK;
}
int afc_sha256_update_batch(afc_ctx* ctx, uint8_t* states, const uint8_t* chunks, const uint64_t* chunk_off, uint32_t n, const uint8_t* final_flags,
                            uint8_t* out32) {
    if (!ctx || !chunk_off || (n && !states)) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    bool any_final = false;
    for (uint32_t i = 0; i < n; i++) {
        if (chunk_off[i + 1] < chunk_off[i]) return AFC_EINVAL;
        const bool fin = final_flags && final_flags[i];
        any_final |= fin;
        if (!fin && ((chunk_off[i + 1] - chunk_off[i]) & 63)) return AFC_EINVAL;      // only a stream's last chunk may be ragged
    }
    if (any_final && !out32) return AFC_EINVAL;
    const uint64_t base = chunk_off[0], bytes = chunk_off[n] - base;
    if (bytes && !chunks) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    std::vector<uint8_t> status(n), dig(any_final ? (size_t)n * 32 : 0);
    Ring ring(ctx, 1);
    RC(ring.once(n, [&](Ring& r) {
        uint8_t *d_chunks, *d_states, *d_fin = nullptr, *d_dig, *d_status;
        const uint64_t* d_off;
        RC(r.stage([&](Stager& k) {
            d_chunks = k.in_at(chunks, base, bytes, 16);
            d_off = k.in(chunk_off, 0, (size_t)n + 1);
            d_states = k.in(states, 0, (size_t)n * AFC_SHA256_STATE_BYTES);
            if (final_flags) d_fin = k.in(final_flags, 0, n);
            d_status = k.take(n);
            d_dig = k.take((size_t)n * 32 + 16);
        }));
        CK(launch::sha256_update(d_states, d_chunks, d_off, n, d_fin, d_dig, d_status, r.st, r.lc));
        return r.copy_back({{states, 0, d_states, (size_t)n * AFC_SHA256_STATE_BYTES}, {status.data(), 0, d_status, n},
                            {dig.data(), 0, d_dig, dig.size()}});
    }));
    for (uint32_t i = 0; i < n; i++) {
        if (!status[i]) return AFC_EINVAL;                                             // a state that is not ours (or not on a block boundary)
        if (final_flags && final_flags[i]) memcpy(out32 + 32ull * i, dig.data() + 32ull * i, 32);
    }
    return AFC_OK;
}
int afc_sha256_update_batch_dev(afc_ctx* ctx, uint8_t* d_states, const uint8_t* d_chunks, const uint64_t* d_chunk_off, uint32_t n,
                                const uint8_t* d_final_flags, uint8_t* d_out32, uint8_t* d_status, void* stream) {
    if (!ctx) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    CallLog lc(ctx);
    CK(launch::sha256_update(d_states, d_chunks, d_chunk_off, n, d_final_flags, d_out32, d_status, (cudaStream_t)stream, lc));
    return AFC_OK;
}

static int expand_common(afc_ctx* ctx, const uint8_t* seeds, uint32_t n, uint8_t* out, size_t item, bool expanded) {
    if (!ctx || (n && (!seeds || !out))) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    CK(cudaSetDevice(ctx->device));
    Ring ring(ctx, 1);
    return ring.once(n, [&](Ring& r) {
        const uint8_t* d_seeds;
        uint8_t* d_out;
        RC(r.stage([&](Stager& k) {
            d_seeds = k.in(seeds, 0, (size_t)n * 32, true);
            d_out = k.take((size_t)n * item, expanded);       // expanded private keys are secret, public keys are not
        }));
        CK(launch::ed_expand_batch(ctx->comb, afc_internal_sign_table(ctx), d_seeds, n, expanded ? d_out : nullptr, expanded ? nullptr : d_out, r.st,
                                   r.lc));
        return r.copy_back({{out, 0, d_out, (size_t)n * item, expanded}});
    });
}
int afc_ed25519_pubkey_batch(afc_ctx* ctx, const uint8_t* seeds, uint32_t n, uint8_t* pks) { return expand_common(ctx, seeds, n, pks, 32, false); }
int afc_ed25519_expand_batch(afc_ctx* ctx, const uint8_t* seeds, uint32_t n, uint8_t* expanded96) { return expand_common(ctx, seeds, n, expanded96, 96, true); }

int afc_ed25519_sign_expanded_batch(afc_ctx* ctx, const uint8_t* expanded96, const uint32_t* key_index, uint32_t n_keys,
                                    const uint8_t* msgs, const uint64_t* msg_off, uint32_t n, uint8_t* sigs) {
    if (!ctx || !msg_off || (n && (!expanded96 || !sigs))) return AFC_EINVAL;
    if (!key_index && n_keys < n) return AFC_EINVAL;
    if (key_index) for (uint32_t i = 0; i < n; i++) if (key_index[i] >= n_keys) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    CK(cudaSetDevice(ctx->device));
    return with_device_keys(ctx, expanded96, n_keys, [&](const uint8_t* d_keys) {
        Ring ring(ctx);
        return ring.walk(n, msg_bytes(msg_off), [&](Ring& r) {
            Msgs M;
            const uint32_t* d_ki = nullptr;
            uint8_t* d_sigs;
            RC(r.stage([&](Stager& k) {
                M = stage_msgs(k, msgs, msg_off, r.i0, r.cnt);
                if (key_index) d_ki = k.in(key_index, r.i0, r.cnt);
                d_sigs = k.take((size_t)r.cnt * 64 + 16);
            }));
            CK(launch::ed_sign_expanded_batch(ctx->comb, afc_internal_sign_table(ctx), d_keys + (key_index ? 0 : (size_t)r.i0 * 96), 0xffffffffu, d_ki,
                                              M.d, M.off, r.cnt, d_sigs, r.st, r.lc));
            return r.copy_back({{sigs, (size_t)r.i0 * 64, d_sigs, (size_t)r.cnt * 64}});
        });
    });
}

// ---------------------------------------------------------------------------------- device-pointer variants
#define DEV_PROLOGUE()                                   \
    if (!ctx) return AFC_EINVAL;                         \
    CK(cudaSetDevice(ctx->device));                      \
    CallLog lc(ctx);                                     \
    cudaStream_t st = (cudaStream_t)stream;
#define DEV_EPILOGUE() return AFC_OK;

int afc_sha256_batch_dev(afc_ctx* ctx, const uint8_t* d_msgs, const uint64_t* d_offsets, uint32_t n, uint8_t* d_out32, void* stream) {
    DEV_PROLOGUE();
    if (!aligned16(d_out32)) return AFC_EINVAL;
    CK(launch::sha256_batch(d_msgs, d_offsets, n, d_out32, st, lc));
    DEV_EPILOGUE();
}
int afc_hmac_sha256_batch_dev(afc_ctx* ctx, const uint8_t* d_keys, const uint32_t* d_key_off, const uint8_t* d_msgs,
                              const uint64_t* d_msg_off, uint32_t n, uint8_t* d_out32, void* stream) {
    DEV_PROLOGUE();
    if (!aligned16(d_out32)) return AFC_EINVAL;
    CK(launch::hmac_sha256_batch(d_keys, d_key_off, d_msgs, d_msg_off, n, d_out32, st, lc));
    DEV_EPILOGUE();
}
int afc_ed25519_verify_batch_dev(afc_ctx* ctx, const uint8_t* d_pks, const uint8_t* d_sigs, const uint8_t* d_msgs,
                                 const uint64_t* d_msg_off, uint32_t n, uint8_t* d_ok, void* stream) {
    DEV_PROLOGUE();
    if (!aligned16(d_pks) || !aligned16(d_sigs)) return AFC_EINVAL;
    // k scratch: per-call allocation from the stream-ordered pool (freed in stream order)
    uint32_t* d_k = nullptr;
    if (n) CK(cudaMallocAsync((void**)&d_k, (size_t)n * 32, st));
    cudaError_t e = verify_with_cache(ctx, d_pks, d_sigs, d_msgs, d_msg_off, n, d_ok, d_k, st, lc);
    if (n) cudaFreeAsync(d_k, st);
    CK(e);
    DEV_EPILOGUE();
}
int afc_ed25519_sign_batch_dev(afc_ctx* ctx, const uint8_t* d_seeds, const uint8_t* d_msgs, const uint64_t* d_msg_off,
                               uint32_t n, uint8_t* d_sigs, void* stream) {
    DEV_PROLOGUE();
    if (!aligned16(d_seeds) || !aligned16(d_sigs)) return AFC_EINVAL;
    CK(launch::ed_sign_batch(ctx->comb, afc_internal_sign_table(ctx), d_seeds, d_msgs, d_msg_off, n, d_sigs, st, lc));
    DEV_EPILOGUE();
}
int afc_ed25519_pubkey_batch_dev(afc_ctx* ctx, const uint8_t* d_seeds, uint32_t n, uint8_t* d_pks, void* stream) {
    DEV_PROLOGUE();
    if (!aligned16(d_seeds) || !aligned16(d_pks)) return AFC_EINVAL;
    CK(launch::ed_expand_batch(ctx->comb, afc_internal_sign_table(ctx), d_seeds, n, nullptr, d_pks, st, lc));
    DEV_EPILOGUE();
}
int afc_ed25519_expand_batch_dev(afc_ctx* ctx, const uint8_t* d_seeds, uint32_t n, uint8_t* d_expanded96, void* stream) {
    DEV_PROLOGUE();
    if (!aligned16(d_seeds) || !aligned16(d_expanded96)) return AFC_EINVAL;
    CK(launch::ed_expand_batch(ctx->comb, afc_internal_sign_table(ctx), d_seeds, n, d_expanded96, nullptr, st, lc));
    DEV_EPILOGUE();
}
int afc_ed25519_sign_expanded_batch_dev(afc_ctx* ctx, const uint8_t* d_expanded96, const uint32_t* d_key_index,
                                        const uint8_t* d_msgs, const uint64_t* d_msg_off, uint32_t n, uint8_t* d_sigs, void* stream) {
    return afc_ed25519_sign_expanded_keys_batch_dev(ctx, d_expanded96, 0xffffffffu, d_key_index, d_msgs, d_msg_off, n, d_sigs, stream);
}
int afc_ed25519_sign_expanded_keys_batch_dev(afc_ctx* ctx, const uint8_t* d_expanded96, uint32_t n_keys, const uint32_t* d_key_index,
                                             const uint8_t* d_msgs, const uint64_t* d_msg_off, uint32_t n, uint8_t* d_sigs, void* stream) {
    DEV_PROLOGUE();
    if (!aligned16(d_expanded96) || !aligned16(d_sigs) || n_keys == 0) return AFC_EINVAL;
    CK(launch::ed_sign_expanded_batch(ctx->comb, afc_internal_sign_table(ctx), d_expanded96, n_keys, d_key_index, d_msgs, d_msg_off, n, d_sigs, st, lc));
    DEV_EPILOGUE();
}
int afc_merkle_leaf_hashes_dev(afc_ctx* ctx, const uint8_t* d_leaves, const uint64_t* d_leaf_off, uint32_t n, uint8_t* d_out32, void* stream) {
    DEV_PROLOGUE();
    if (!aligned16(d_out32)) return AFC_EINVAL;
    CK(launch::merkle_leaf_hashes(d_leaves, d_leaf_off, n, d_out32, st, lc));
    DEV_EPILOGUE();
}


int afc_b64url_encode_fixed_dev(afc_ctx* ctx, const uint8_t* d_in, uint32_t item_bytes, uint32_t n, uint8_t* d_out, void* stream) {
    DEV_PROLOGUE();
    if (n && item_bytes && (!d_in || !d_out)) return AFC_EINVAL;
    CK(launch::b64url_encode(d_in, item_bytes, n, d_out, st, lc));
    DEV_EPILOGUE();
}
int afc_hex_encode_fixed_dev(afc_ctx* ctx, const uint8_t* d_in, uint32_t item_bytes, uint32_t n, uint8_t* d_out, void* stream) {
    DEV_PROLOGUE();
    if (n && item_bytes && (!d_in || !d_out)) return AFC_EINVAL;
    CK(launch::hex_encode(d_in, (uint64_t)item_bytes * n, d_out, st, lc));
    DEV_EPILOGUE();
}


int afc_json_fill_sizes_dev(afc_ctx* ctx, const uint8_t* d_segs, const uint32_t* d_seg_off, const uint8_t* d_kinds, uint32_t n_fields,
                            const uint8_t* d_fields, const uint64_t* d_field_off, uint32_t n, uint64_t* d_out_off, uint64_t* total_bytes, void* stream) {
    DEV_PROLOGUE();
    if (!d_seg_off || !d_out_off || (n_fields && !d_kinds) || (n && n_fields && !d_field_off)) return AFC_EINVAL;
    uint64_t* d_scratch = nullptr;
    CK(cudaMallocAsync((void**)&d_scratch, launch::json_scan_scratch_bytes(n), st));
    cudaError_t e = launch::json_fill_sizes(d_segs, d_seg_off, d_kinds, n_fields, d_fields, d_field_off, n, d_out_off, d_scratch, st, lc);
    cudaFreeAsync(d_scratch, st);
    CK(e);
    if (total_bytes) {
        CK(cudaMemcpyAsync(total_bytes, d_out_off + n, 8, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    DEV_EPILOGUE();
}
int afc_json_fill_dev(afc_ctx* ctx, const uint8_t* d_segs, const uint32_t* d_seg_off, const uint8_t* d_kinds, uint32_t n_fields,
                      const uint8_t* d_fields, const uint64_t* d_field_off, uint32_t n, const uint64_t* d_out_off, uint8_t* d_out, void* stream) {
    DEV_PROLOGUE();
    if (!d_seg_off || !d_out_off || (n && !d_out) || (n_fields && !d_kinds) || (n && n_fields && !d_field_off)) return AFC_EINVAL;
    CK(launch::json_fill(d_segs, d_seg_off, d_kinds, n_fields, d_fields, d_field_off, n, d_out_off, d_out, st, lc));
    DEV_EPILOGUE();
}


int afc_keycache_configure(afc_ctx* ctx, uint32_t max_keys) {
    if (!ctx) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(ctx->kc_mu);
    CK(cudaDeviceSynchronize());
    kc_free(ctx);
    ctx->kc_max_keys = max_keys;
    return AFC_OK;
}
int afc_keycache_clear(afc_ctx* ctx, void* stream) {
    if (!ctx) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(ctx->kc_mu);
    if (!ctx->kc_ready) return AFC_OK;
    cudaStream_t st = (cudaStream_t)stream;
    CK(cudaStreamWaitEvent(st, ctx->kc_event, 0));
    {
        CallLog lc(ctx);
        CK(launch::ed_keycache_clear(ctx->kc, st, lc));
    }
    CK(cudaEventRecord(ctx->kc_event, st));
    return AFC_OK;
}
static int kc_read_state(afc_ctx* ctx, uint32_t* st) {
    memset(st, 0, launch::KS_WORDS * 4);
    if (ctx->kc_ready) { CK(cudaDeviceSynchronize()); CK(cudaMemcpy(st, ctx->kc.state, launch::KS_WORDS * 4, cudaMemcpyDeviceToHost)); }
    return AFC_OK;
}
int afc_keycache_info(afc_ctx* ctx, uint32_t* max_keys, uint32_t* cached_keys, uint32_t* last_mode) {
    if (!ctx) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(ctx->kc_mu);
    uint32_t st[launch::KS_WORDS];
    int rc = kc_read_state(ctx, st);
    if (rc != AFC_OK) return rc;
    if (max_keys) *max_keys = ctx->kc_max_keys;
    if (cached_keys) *cached_keys = st[launch::KS_HIGH] - st[launch::KS_NFREE];
    if (last_mode) *last_mode = st[launch::KS_NHOT] ? 1u : 0u;
    return AFC_OK;
}
int afc_keycache_stats(afc_ctx* ctx, afc_keycache_stats_t* out) {
    if (!ctx || !out) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(ctx->kc_mu);
    uint32_t st[launch::KS_WORDS];
    int rc = kc_read_state(ctx, st);
    if (rc != AFC_OK) return rc;
    out->max_keys = ctx->kc_max_keys; out->cached_keys = st[launch::KS_HIGH] - st[launch::KS_NFREE];
    out->last_hot = st[launch::KS_NHOT]; out->last_cold = st[launch::KS_NCOLD]; out->last_distinct = st[launch::KS_DISTINCT];
    out->last_built = st[launch::KS_NBUILD]; out->last_evicted = st[launch::KS_EVICTED];
    out->total_built = st[launch::KS_TOTAL_BUILT]; out->total_evicted = st[launch::KS_TOTAL_EVICTED]; out->calls = st[launch::KS_CALLS];
    return AFC_OK;
}

// ---------------------------------------------------------------------------------- keyed verification
int afc_keyset_new(afc_ctx* ctx, const uint8_t* pks, uint32_t n_keys, afc_keyset** out) {
    if (!ctx || !out || !pks || n_keys == 0) return AFC_EINVAL;
    *out = nullptr;
    CK(cudaSetDevice(ctx->device));
    afc_keyset* ks = new (std::nothrow) afc_keyset();
    if (!ks) return AFC_ENOMEM;
    ks->ctx = ctx; ks->n_keys = n_keys; ks->tab_bytes = launch::ed_key_table_bytes(n_keys);
    cudaError_t e = cudaMalloc((void**)&ks->d_pks, (size_t)n_keys * 32);
    if (e == cudaSuccess) e = cudaMalloc((void**)&ks->d_valid, n_keys);
    if (e == cudaSuccess) e = cudaMalloc(&ks->d_tabs, ks->tab_bytes);
    if (e == cudaSuccess) e = cudaMemcpy(ks->d_pks, pks, (size_t)n_keys * 32, cudaMemcpyHostToDevice);
    void* d_bases = nullptr;
    if (e == cudaSuccess) e = cudaMalloc(&d_bases, launch::ed_key_bases_bytes(n_keys));
    if (e == cudaSuccess) {
        CallLog lc(ctx);
        e = launch::ed_build_key_tables(ks->d_pks, n_keys, ks->d_tabs, ks->d_valid, d_bases, 0, lc);
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
    }
    if (d_bases) cudaFree(d_bases);
    if (e != cudaSuccess) {
        set_err(ctx, e, "afc_keyset_new");
        afc_keyset_free(ks);
        return e == cudaErrorMemoryAllocation ? AFC_ENOMEM : AFC_ECUDA;
    }
    *out = ks;
    return AFC_OK;
}
void afc_keyset_free(afc_keyset* ks) {
    if (!ks) return;
    cudaSetDevice(ks->ctx->device);
    if (ks->d_pks) cudaFree(ks->d_pks);
    if (ks->d_valid) cudaFree(ks->d_valid);
    if (ks->d_tabs) cudaFree(ks->d_tabs);
    void* named[] = {ks->d_dids, ks->d_did_off, ks->d_slots, ks->d_schemas, ks->d_vcj_schemas};
    for (void* p : named) if (p) cudaFree(p);
    delete ks;
}
int afc_keyset_info(afc_keyset* ks, uint32_t* n_keys, uint64_t* table_bytes) {
    if (!ks) return AFC_EINVAL;
    if (n_keys) *n_keys = ks->n_keys;
    if (table_bytes) *table_bytes = ks->tab_bytes;
    return AFC_OK;
}
int afc_ed25519_verify_keyed_batch(afc_ctx* ctx, afc_keyset* ks, const uint32_t* key_index, const uint8_t* sigs,
                                   const uint8_t* msgs, const uint64_t* msg_off, uint32_t n, uint8_t* ok) {
    if (!ctx || !ks || ks->ctx != ctx || !msg_off || (n && (!key_index || !sigs || !ok))) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    CK(cudaSetDevice(ctx->device));
    Ring ring(ctx);
    return ring.walk(n, msg_bytes(msg_off), [&](Ring& r) {
        Msgs M;
        const uint32_t* d_ki;
        const uint8_t* d_sigs;
        uint8_t* d_ok;
        uint32_t* d_k;
        RC(r.stage([&](Stager& k) {
            M = stage_msgs(k, msgs, msg_off, r.i0, r.cnt);
            d_sigs = k.in(sigs, (size_t)r.i0 * 64, (size_t)r.cnt * 64);
            d_ki = k.in(key_index, r.i0, r.cnt);
            d_ok = k.take((size_t)r.cnt + 16);
            d_k = (uint32_t*)k.take((size_t)r.cnt * 32 + launch::ed_keyed_scratch_bytes(ks->n_keys, r.cnt));
        }));
        CK(launch::ed_verify_keyed_batch(ctx->comb, ks->d_tabs, ks->d_valid, ks->d_pks, ks->n_keys, d_ki, d_sigs, M.d, M.off, r.cnt, d_ok, d_k,
                                         d_k + (size_t)r.cnt * 8, r.st, r.lc));
        return r.copy_back({{ok, r.i0, d_ok, r.cnt}});
    });
}
int afc_ed25519_verify_keyed_batch_dev(afc_ctx* ctx, afc_keyset* ks, const uint32_t* d_key_index, const uint8_t* d_sigs,
                                       const uint8_t* d_msgs, const uint64_t* d_msg_off, uint32_t n, uint8_t* d_ok, void* stream) {
    if (!ctx || !ks || ks->ctx != ctx) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    if (!aligned16(d_sigs)) return AFC_EINVAL;
    CallLog lc(ctx);
    cudaStream_t st = (cudaStream_t)stream;
    uint32_t* d_k = nullptr;
    if (n) CK(cudaMallocAsync((void**)&d_k, (size_t)n * 32 + launch::ed_keyed_scratch_bytes(ks->n_keys, n), st));
    cudaError_t e = launch::ed_verify_keyed_batch(ctx->comb, ks->d_tabs, ks->d_valid, ks->d_pks, ks->n_keys, d_key_index, d_sigs, d_msgs,
                                                  d_msg_off, n, d_ok, d_k, n ? d_k + (size_t)n * 8 : nullptr, st, lc);
    if (n) cudaFreeAsync(d_k, st);
    CK(e);
    return AFC_OK;
}

// ---------------------------------------------------------------------------------- stored credential documents
static uint32_t did_hash(const uint8_t* p, uint64_t n) {
    uint32_t h = 2166136261u;
    for (uint64_t j = 0; j < n; j++) h = (h ^ p[j]) * 16777619u;          // = vc_did_hash_byte (afc_vcdoc.cuh)
    return h;
}
int afc_keyset_new_named(afc_ctx* ctx, const uint8_t* pks, const uint8_t* dids, const uint64_t* did_off, uint32_t n_keys, afc_keyset** out) {
    if (!ctx || !out || !pks || !dids || !did_off || n_keys == 0) return AFC_EINVAL;
    *out = nullptr;
    const uint64_t base = did_off[0], total = did_off[n_keys] - base;
    for (uint32_t k = 0; k < n_keys; k++) if (did_off[k + 1] < did_off[k]) return AFC_EINVAL;
    if (total >= 0xffffffffull) return AFC_EINVAL;
    uint32_t cap = 2; while (cap < 2ull * n_keys) cap <<= 1;
    std::vector<uint32_t> slots(cap, 0xffffffffu), off(n_keys + 1);
    for (uint32_t k = 0; k <= n_keys; k++) off[k] = (uint32_t)(did_off[k] - base);
    for (uint32_t k = 0; k < n_keys; k++) {
        const uint8_t* d = dids + did_off[k];
        const uint64_t len = did_off[k + 1] - did_off[k];
        uint32_t s = did_hash(d, len) & (cap - 1);
        for (; slots[s] != 0xffffffffu; s = (s + 1) & (cap - 1)) {
            const uint32_t o = slots[s];
            if (did_off[o + 1] - did_off[o] == len && memcmp(dids + did_off[o], d, len) == 0) return AFC_EINVAL;     // duplicate DID
        }
        slots[s] = k;
    }
    int rc = afc_keyset_new(ctx, pks, n_keys, out);
    if (rc != AFC_OK) return rc;
    afc_keyset* ks = *out;
    ks->slot_mask = cap - 1;
    const size_t sb = launch::vc_schema_bytes();
    std::vector<uint8_t> schemas(2 * sb);
    const size_t jb = launch::vcj_schema_bytes();
    std::vector<uint8_t> jschemas(2 * jb);
    if (launch::vc_schema_host(0, schemas.data()) != 0 || launch::vc_schema_host(1, schemas.data() + sb) != 0 ||
        launch::vcj_schema_host(0, jschemas.data()) != 0 || launch::vcj_schema_host(1, jschemas.data() + jb) != 0) {
        afc_keyset_free(ks); *out = nullptr; return AFC_EINVAL;
    }
    cudaError_t e = cudaMalloc((void**)&ks->d_dids, total + 4);
    if (e == cudaSuccess) e = cudaMalloc((void**)&ks->d_did_off, ((size_t)n_keys + 1) * 4);
    if (e == cudaSuccess) e = cudaMalloc((void**)&ks->d_slots, (size_t)cap * 4);
    if (e == cudaSuccess) e = cudaMalloc((void**)&ks->d_schemas, 2 * sb);
    if (e == cudaSuccess) e = cudaMalloc((void**)&ks->d_vcj_schemas, 2 * jb);
    if (e == cudaSuccess && total) e = cudaMemcpy(ks->d_dids, dids + base, total, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(ks->d_did_off, off.data(), ((size_t)n_keys + 1) * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(ks->d_slots, slots.data(), (size_t)cap * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(ks->d_schemas, schemas.data(), 2 * sb, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(ks->d_vcj_schemas, jschemas.data(), 2 * jb, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        set_err(ctx, e, "afc_keyset_new_named");
        afc_keyset_free(ks); *out = nullptr;
        return e == cudaErrorMemoryAllocation ? AFC_ENOMEM : AFC_ECUDA;
    }
    ks->named = true;
    return AFC_OK;
}
static int vc_stored_check(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, uint8_t* status) {
    if (!ctx || !ks || ks->ctx != ctx || !doc_off || (n && (!docs || !status))) return AFC_EINVAL;
    if (doc_kind != AFC_DOC_EXECUTION_VC && doc_kind != AFC_DOC_WORKFLOW_VC) return AFC_EINVAL;
    if (!ks->named) return AFC_ESTATE;
    return AFC_OK;
}
// the host-buffer form of afc_vc_verify_stored_batch (json = false) and afc_vc_verify_json_batch (json = true)
static int vc_verify_host(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, uint8_t* status,
                          uint32_t* fields, bool json) {
    int rc = vc_stored_check(ctx, ks, doc_kind, docs, doc_off, n, status);
    if (rc != AFC_OK || n == 0) return rc;
    CK(cudaSetDevice(ctx->device));
    Ring ring(ctx);
    return ring.walk(n, msg_bytes(doc_off), [&](Ring& r) {
        Msgs D;
        uint8_t* d_status;
        uint32_t* d_fields = nullptr;
        VcScratch S;
        RC(r.stage([&](Stager& k) {
            D = stage_msgs(k, docs, doc_off, r.i0, r.cnt);
            d_status = k.take((size_t)r.cnt + 16);
            if (fields) d_fields = k.take<uint32_t>((size_t)r.cnt * 4 + 4);
            vc_scratch(k, S, r.cnt, doc_off[r.i0 + r.cnt] - doc_off[r.i0], ks->n_keys, false);
        }));
        CK(vc_stored_enqueue(ctx, ks, doc_kind, D.d, D.off, r.cnt, d_status, d_fields, S, r.st, r.lc, nullptr, nullptr, nullptr, json));
        return r.copy_back({{status, r.i0, d_status, r.cnt}, {fields, (size_t)r.i0 * 16, d_fields, fields ? (size_t)r.cnt * 16 : 0}});
    });
}
int afc_vc_verify_stored_batch(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* docs, const uint64_t* doc_off, uint32_t n,
                               uint8_t* status, uint32_t* fields) {
    return vc_verify_host(ctx, ks, doc_kind, docs, doc_off, n, status, fields, false);
}
// the _dev form of afc_vc_verify_stored_batch (json = false) and afc_vc_verify_json_batch (json = true)
static int vc_verify_dev(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* d_docs, const uint64_t* d_doc_off, uint32_t n, uint8_t* d_status,
                         uint32_t* d_fields, void* stream, bool json) {
    int rc = vc_stored_check(ctx, ks, doc_kind, d_docs, d_doc_off, n, d_status);
    if (rc != AFC_OK || n == 0) return rc;
    if (d_fields && !aligned16(d_fields)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    CallLog lc(ctx);
    cudaStream_t st = (cudaStream_t)stream;
    uint64_t ends[2];                       // the batch's byte size bounds the message buffer: read it once (one synchronisation)
    CK(cudaMemcpyAsync(&ends[0], d_doc_off, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&ends[1], d_doc_off + n, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (ends[1] < ends[0]) return AFC_EINVAL;
    uint8_t* scratch = nullptr;
    VcScratch S;
    CK(pool_carve(&scratch, st, [&](Carve& k) { vc_scratch(k, S, n, ends[1] - ends[0], ks->n_keys, false); }));
    cudaError_t e = vc_stored_enqueue(ctx, ks, doc_kind, d_docs, d_doc_off, n, d_status, d_fields, S, st, lc, nullptr, nullptr, nullptr, json);
    cudaFreeAsync(scratch, st);
    CK(e);
    return AFC_OK;
}
int afc_vc_verify_stored_batch_dev(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* d_docs, const uint64_t* d_doc_off, uint32_t n,
                                   uint8_t* d_status, uint32_t* d_fields, void* stream) {
    return vc_verify_dev(ctx, ks, doc_kind, d_docs, d_doc_off, n, d_status, d_fields, stream, false);
}

// documents in any JSON spelling: the arguments, statuses and fields of afc_vc_verify_stored_batch
int afc_vc_verify_json_batch(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* docs, const uint64_t* doc_off, uint32_t n,
                             uint8_t* status, uint32_t* fields) {
    return vc_verify_host(ctx, ks, doc_kind, docs, doc_off, n, status, fields, true);
}
int afc_vc_verify_json_batch_dev(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* d_docs, const uint64_t* d_doc_off, uint32_t n,
                                 uint8_t* d_status, uint32_t* d_fields, void* stream) {
    return vc_verify_dev(ctx, ks, doc_kind, d_docs, d_doc_off, n, d_status, d_fields, stream, true);
}

// audit: the arguments of afc_vc_verify_stored_batch, plus columns exactly for execution documents
static int vc_audit_check(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* docs, const uint64_t* doc_off, const uint8_t* cols,
                          const uint64_t* col_off, uint32_t n, uint8_t* status, uint32_t* issues) {
    int rc = vc_stored_check(ctx, ks, doc_kind, docs, doc_off, n, status);
    if (rc != AFC_OK && rc != AFC_ESTATE) return rc;
    if (n && !issues) return AFC_EINVAL;
    if (doc_kind == AFC_DOC_EXECUTION_VC ? (!col_off || (n && !cols)) : (cols || col_off)) return AFC_EINVAL;
    return rc;
}
int afc_vc_audit_stored_batch(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* docs, const uint64_t* doc_off, const uint8_t* cols,
                              const uint64_t* col_off, uint32_t n, uint8_t* status, uint32_t* issues) {
    int rc = vc_audit_check(ctx, ks, doc_kind, docs, doc_off, cols, col_off, n, status, issues);
    if (rc != AFC_OK || n == 0) return rc;
    const uint32_t C = AFC_AUDIT_COLUMNS;
    CK(cudaSetDevice(ctx->device));
    Ring ring(ctx);
    auto measure = [&](uint32_t i0, uint32_t i) {
        if (col_off) for (uint32_t k = 0; k < C; k++) if (col_off[(size_t)i * C + k + 1] < col_off[(size_t)i * C + k]) return kBadOffsets;
        return msg_bytes(doc_off)(i0, i);
    };
    return ring.walk(n, measure, [&](Ring& r) {
        Msgs D;
        const uint8_t* d_cols = nullptr;
        const uint64_t* d_coff = nullptr;
        uint8_t* d_status;
        uint32_t* d_issues;
        VcScratch S;
        RC(r.stage([&](Stager& k) {
            D = stage_msgs(k, docs, doc_off, r.i0, r.cnt);
            if (col_off) {
                const uint64_t cbase = col_off[(size_t)r.i0 * C];
                d_cols = k.in_at(cols, cbase, col_off[(size_t)(r.i0 + r.cnt) * C] - cbase, 16);
                d_coff = k.in(col_off, (size_t)r.i0 * C, (size_t)r.cnt * C + 1);
            }
            d_status = k.take((size_t)r.cnt + 16);
            d_issues = k.take<uint32_t>((size_t)r.cnt + 4);
            vc_scratch(k, S, r.cnt, doc_off[r.i0 + r.cnt] - doc_off[r.i0], ks->n_keys, true);
        }));
        CK(vc_stored_enqueue(ctx, ks, doc_kind, D.d, D.off, r.cnt, d_status, nullptr, S, r.st, r.lc, d_issues, d_cols, d_coff));
        return r.copy_back({{status, r.i0, d_status, r.cnt}, {issues, (size_t)r.i0 * 4, d_issues, (size_t)r.cnt * 4}});
    });
}
int afc_vc_audit_stored_batch_dev(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* d_docs, const uint64_t* d_doc_off, const uint8_t* d_cols,
                                  const uint64_t* d_col_off, uint32_t n, uint8_t* d_status, uint32_t* d_issues, void* stream) {
    int rc = vc_audit_check(ctx, ks, doc_kind, d_docs, d_doc_off, d_cols, d_col_off, n, d_status, d_issues);
    if (rc != AFC_OK || n == 0) return rc;
    CK(cudaSetDevice(ctx->device));
    CallLog lc(ctx);
    cudaStream_t st = (cudaStream_t)stream;
    uint64_t ends[2];                       // the batch's byte size bounds the message buffer: read it once (one synchronisation)
    CK(cudaMemcpyAsync(&ends[0], d_doc_off, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&ends[1], d_doc_off + n, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (ends[1] < ends[0]) return AFC_EINVAL;
    uint8_t* scratch = nullptr;
    VcScratch S;
    CK(pool_carve(&scratch, st, [&](Carve& k) { vc_scratch(k, S, n, ends[1] - ends[0], ks->n_keys, true); }));
    cudaError_t e = vc_stored_enqueue(ctx, ks, doc_kind, d_docs, d_doc_off, n, d_status, nullptr, S, st, lc, d_issues, d_cols, d_col_off);
    cudaFreeAsync(scratch, st);
    CK(e);
    return AFC_OK;
}

// ---------------------------------------------------------------------------------- issuing execution credentials
// Bounds from the column bytes alone (so that the _dev call needs nothing but the two ends of col_off): each credential's constant
// text, four digests, a 20-character int64, the 86 proofValue characters and the errorMessage member's frame and suffix, plus at
// most 6 bytes per column byte (backslash-u 00XX, or backslash-u fffd for an invalid byte) for each of its at most 3 appearances in the stored document
// (caller_did: issuer, caller.did, verificationMethod) and 2 in the signing message.
static uint64_t issue_fixed_bytes() { return launch::vci_literal_bytes() + 4 * 43 + 20 + 86 + 32; }
static uint64_t issue_doc_bound(uint32_t n, uint64_t col_bytes) { return (uint64_t)n * issue_fixed_bytes() + 18 * col_bytes; }
static uint64_t issue_msg_bound(uint32_t n, uint64_t col_bytes) { return (uint64_t)n * issue_fixed_bytes() + 12 * col_bytes; }

uint64_t afc_vc_issue_bound(const uint64_t* col_off, uint32_t n) {
    if (!col_off || n == 0) return 0;
    const uint64_t a = col_off[0], b = col_off[(size_t)n * AFC_ISSUE_COLUMNS];
    return issue_doc_bound(n, b >= a ? b - a : 0);
}

// per-call device scratch: signing messages and their offsets, signatures, scan tiles
struct IssueScratch { uint8_t* msgs; uint64_t* msg_off; uint8_t* sigs; uint64_t* scan; };
static void issue_scratch(Carve& k, IssueScratch& s, uint32_t n, uint64_t col_bytes) {
    s.msgs = k.take(issue_msg_bound(n, col_bytes) + 64);
    s.msg_off = k.take<uint64_t>((size_t)n + 1);
    s.sigs = k.take((size_t)n * 64);
    s.scan = (uint64_t*)k.take(launch::json_scan_scratch_bytes(n));
}
// hashData, both lengths, both scans: doc_off is complete when this has run
static cudaError_t issue_sizes(const uint8_t* cols, const uint64_t* col_off, const int64_t* dur, const uint8_t* pay, const uint64_t* pay_off,
                               const uint8_t* nil, uint8_t* hashes, uint32_t n, uint64_t* doc_off, const IssueScratch& S, cudaStream_t st,
                               launch::LaunchLog* lg) {
    cudaError_t e = hashes ? launch::vci_hashdata(pay, pay_off, nil, 2 * n, hashes, st, lg) : cudaSuccess;
    if (e == cudaSuccess) e = launch::vci_sizes(cols, col_off, dur, hashes, n, S.msg_off + 1, doc_off + 1, st, lg);
    if (e == cudaSuccess) e = launch::offsets_from_lengths(S.msg_off, n, S.scan, st, lg);
    if (e == cudaSuccess) e = launch::offsets_from_lengths(doc_off, n, S.scan, st, lg);
    return e;
}
// both byte strings, the signatures, the proofValues
static cudaError_t issue_finish(afc_ctx* ctx, const uint8_t* d_exp, uint32_t n_keys, const uint32_t* key_index, const uint8_t* cols,
                                const uint64_t* col_off, const int64_t* dur, const uint8_t* hashes, uint32_t n, uint8_t* docs, const uint64_t* doc_off,
                                uint8_t* pv, const IssueScratch& S, cudaStream_t st, launch::LaunchLog* lg) {
    cudaError_t e = launch::vci_fill(cols, col_off, dur, hashes, n, S.msg_off, S.msgs, doc_off, docs, st, lg);
    if (e == cudaSuccess) e = launch::ed_sign_expanded_batch(ctx->comb, afc_internal_sign_table(ctx), d_exp, n_keys, key_index, S.msgs, S.msg_off, n,
                                                             S.sigs, st, lg);
    if (e == cudaSuccess) e = launch::vci_proof(S.sigs, n, doc_off, docs, pv, st, lg);
    return e;
}
static int issue_check(afc_ctx* ctx, const uint8_t* expanded96, uint32_t n_keys, const uint32_t* key_index, const uint8_t* cols,
                       const uint64_t* col_off, const int64_t* duration_ms, const uint8_t* payloads, const uint64_t* payload_off,
                       const uint8_t* payload_nil, uint32_t flags, uint32_t n, afc_merkle* log, const uint8_t* docs, const uint64_t* doc_off,
                       const uint8_t* hashes, const uint8_t* proof_values) {
    if (!ctx || !col_off || !doc_off || (flags & ~(uint32_t)AFC_ISSUE_HASH_DATA)) return AFC_EINVAL;
    if (log && log->ctx != ctx) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    if (!expanded96 || n_keys == 0 || !key_index || !cols || !duration_ms || !docs || !proof_values) return AFC_EINVAL;
    if ((flags & AFC_ISSUE_HASH_DATA) && (!hashes || !payloads || !payload_off || !payload_nil)) return AFC_EINVAL;
    return AFC_OK;
}

int afc_vc_issue_execution_batch_dev(afc_ctx* ctx, const uint8_t* d_expanded96, uint32_t n_keys, const uint32_t* d_key_index, const uint8_t* d_cols,
                                     const uint64_t* d_col_off, const int64_t* d_duration_ms, const uint8_t* d_payloads,
                                     const uint64_t* d_payload_off, const uint8_t* d_payload_nil, uint32_t flags, uint32_t n, afc_merkle* log,
                                     uint8_t* d_docs, uint64_t docs_cap, uint64_t* d_doc_off, uint8_t* d_hashes, uint8_t* d_proof_values,
                                     void* stream) {
    int rc = issue_check(ctx, d_expanded96, n_keys, d_key_index, d_cols, d_col_off, d_duration_ms, d_payloads, d_payload_off, d_payload_nil, flags,
                         n, log, d_docs, d_doc_off, d_hashes, d_proof_values);
    if (rc != AFC_OK || n == 0) return rc;
    if (!aligned16(d_expanded96)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    uint64_t ends[2];                       // the column bytes bound the documents: read them once (one synchronisation)
    CK(cudaMemcpyAsync(&ends[0], d_col_off, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&ends[1], d_col_off + (size_t)n * AFC_ISSUE_COLUMNS, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (ends[1] < ends[0] || docs_cap < issue_doc_bound(n, ends[1] - ends[0])) return AFC_EINVAL;
    const uint64_t cb = ends[1] - ends[0];
    uint8_t* hashes = (flags & AFC_ISSUE_HASH_DATA) ? d_hashes : nullptr;
    {
        CallLog lc(ctx);
        uint8_t* scratch = nullptr;
        IssueScratch S;
        CK(pool_carve(&scratch, st, [&](Carve& k) { issue_scratch(k, S, n, cb); }));
        cudaError_t e = issue_sizes(d_cols, d_col_off, d_duration_ms, d_payloads, d_payload_off, d_payload_nil, hashes, n, d_doc_off, S, st, lc);
        if (e == cudaSuccess) e = issue_finish(ctx, d_expanded96, n_keys, d_key_index, d_cols, d_col_off, d_duration_ms, hashes, n, d_docs, d_doc_off,
                                               d_proof_values, S, st, lc);
        cudaFreeAsync(scratch, st);
        CK(e);
    }
    return log ? afc_merkle_append_dev(log, d_docs, d_doc_off, n, stream) : AFC_OK;
}

int afc_vc_issue_execution_batch(afc_ctx* ctx, const uint8_t* expanded96, uint32_t n_keys, const uint32_t* key_index, const uint8_t* cols,
                                 const uint64_t* col_off, const int64_t* duration_ms, const uint8_t* payloads, const uint64_t* payload_off,
                                 const uint8_t* payload_nil, uint32_t flags, uint32_t n, afc_merkle* log, uint8_t* docs, uint64_t docs_cap,
                                 uint64_t* doc_off, uint8_t* hashes, uint8_t* proof_values) {
    int rc = issue_check(ctx, expanded96, n_keys, key_index, cols, col_off, duration_ms, payloads, payload_off, payload_nil, flags, n, log, docs,
                         doc_off, hashes, proof_values);
    if (rc != AFC_OK) return rc;
    if (n == 0) { doc_off[0] = 0; return AFC_OK; }
    const bool hash = (flags & AFC_ISSUE_HASH_DATA) != 0;
    for (uint32_t i = 0; i < n; i++) if (key_index[i] >= n_keys) return AFC_EINVAL;
    uint64_t bad = 0;
    for (size_t k = 0; k < (size_t)n * AFC_ISSUE_COLUMNS; k++) bad |= (uint64_t)(col_off[k + 1] < col_off[k]);
    if (hash) for (size_t k = 0; k < (size_t)2 * n; k++) bad |= (uint64_t)(payload_off[k + 1] < payload_off[k]);
    if (bad || docs_cap < afc_vc_issue_bound(col_off, n)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    // Chunks of credentials through the ring.  A chunk's documents land at their final offsets, so its stream is synchronised once after
    // the sizes pass to learn where the chunk ends (the next chunk's copies are enqueued after that).
    const uint32_t C = AFC_ISSUE_COLUMNS;
    auto measure = [&](uint32_t i0, uint32_t i) {
        return (col_off[(size_t)(i + 1) * C] - col_off[(size_t)i0 * C]) + (hash ? payload_off[2 * (size_t)(i + 1)] - payload_off[2 * (size_t)i0] : 0);
    };
    uint64_t base = 0;
    return with_device_keys(ctx, expanded96, n_keys, [&](const uint8_t* d_keys) {
        Ring ring(ctx);
        return ring.walk(n, measure, [&](Ring& r) {
            const uint32_t i0 = r.i0, cnt = r.cnt;
            const uint64_t cbase = col_off[(size_t)i0 * C], cbytes = col_off[(size_t)(i0 + cnt) * C] - cbase;
            const uint64_t pbase = hash ? payload_off[2 * (size_t)i0] : 0, pbytes = hash ? payload_off[2 * (size_t)(i0 + cnt)] - pbase : 0;
            const uint8_t *d_cols, *d_pay = nullptr, *d_nil = nullptr;
            const uint64_t *d_coff, *d_poff = nullptr;
            const int64_t* d_dur;
            const uint32_t* d_ki;
            uint8_t *d_docs, *d_h = nullptr, *d_pv;
            uint64_t* d_doff;
            IssueScratch S;
            RC(r.stage([&](Stager& k) {
                d_cols = k.in_at(cols, cbase, cbytes, 16);
                d_coff = k.in(col_off, (size_t)i0 * C, (size_t)cnt * C + 1);
                d_dur = k.in(duration_ms, i0, cnt);
                d_ki = k.in(key_index, i0, cnt);
                if (hash) {
                    d_pay = k.in_at(payloads, pbase, pbytes, 16);
                    d_poff = k.in(payload_off, 2 * (size_t)i0, 2 * (size_t)cnt + 1);
                    d_nil = k.in(payload_nil, 2 * (size_t)i0, 2 * (size_t)cnt);
                    d_h = k.take((size_t)cnt * 86);
                }
                d_docs = k.take(issue_doc_bound(cnt, cbytes) + 64);
                d_doff = k.take<uint64_t>((size_t)cnt + 1);
                d_pv = k.take((size_t)cnt * 86);
                issue_scratch(k, S, cnt, cbytes);
            }));
            CK(issue_sizes(d_cols, d_coff, d_dur, d_pay, d_poff, d_nil, d_h, cnt, d_doff, S, r.st, r.lc));
            uint64_t bytes;
            RC(r.read(&bytes, {d_doff + cnt}));
            CK(issue_finish(ctx, d_keys, n_keys, d_ki, d_cols, d_coff, d_dur, d_h, cnt, d_docs, d_doff, d_pv, S, r.st, r.lc));
            RC(r.copy_back({offsets_out(doc_off, i0, d_doff, (size_t)cnt + 1, base), {hashes, (size_t)i0 * 86, d_h, hash ? (size_t)cnt * 86 : 0},
                            {proof_values, (size_t)i0 * 86, d_pv, (size_t)cnt * 86}, {docs, base, d_docs, bytes}}));
            if (log) RC(afc_merkle_append_dev(log, d_docs, d_doff, cnt, r.st));
            base += bytes;
            return AFC_OK;
        });
    });
}

// ---------------------------------------------------------------------------------- issuing workflow credentials
// Bounds from the three offset arrays' ends alone: each workflow's constant text, three counts of at most 10 digits, the longest status
// name, startTime, the endTime member, the array's brackets and the 86 proofValue characters; at most 6 bytes per column byte for each of
// its at most 4 appearances in the stored document (issuer_did: issuer, orchestrator.did and agentNodeDid, verificationMethod), and per
// record its escaped id in quotes with a comma.  The signing message never holds more than the stored document.
static uint64_t wf_fixed_bytes() { return launch::vcw_literal_bytes() + 3 * 10 + 9 + 20 + 33 + 2 + 86; }
static uint64_t wf_doc_bound(uint32_t n, uint64_t col_bytes, uint64_t records, uint64_t rec_bytes) {
    return (uint64_t)n * wf_fixed_bytes() + 24 * col_bytes + 6 * rec_bytes + 3 * records;
}

uint64_t afc_vc_workflow_bound(const uint64_t* col_off, const uint64_t* rec_off, const uint64_t* rec_col_off, uint32_t n) {
    if (!col_off || !rec_off || !rec_col_off || n == 0) return 0;
    const uint64_t a = col_off[0], b = col_off[(size_t)n * AFC_WORKFLOW_COLUMNS], r0 = rec_off[0], r1 = rec_off[n];
    if (r1 < r0) return wf_doc_bound(n, b >= a ? b - a : 0, 0, 0);
    const uint64_t c = rec_col_off[2 * r0], d = rec_col_off[2 * r1];
    return wf_doc_bound(n, b >= a ? b - a : 0, r1 - r0, d >= c ? d - c : 0);
}

// per-call device scratch: signing messages and their offsets, signatures, scan tiles, record classes, record id offsets, array places
struct WorkflowScratch { uint8_t* msgs; uint64_t* msg_off; uint8_t* sigs; uint64_t* scan; uint8_t* cls; uint64_t* id_off; uint64_t* arr; };
static void wf_scratch(Carve& k, WorkflowScratch& s, uint32_t n, uint32_t m, uint64_t msg_bound) {
    s.msgs = k.take(msg_bound + 64);
    s.msg_off = k.take<uint64_t>((size_t)n + 1);
    s.sigs = k.take((size_t)n * 64);
    s.scan = (uint64_t*)k.take(launch::json_scan_scratch_bytes(n > m ? n : m));
    s.cls = k.take(m);
    s.id_off = k.take<uint64_t>((size_t)m + 1);
    s.arr = k.take<uint64_t>((size_t)n * 2);
}
// records, plans and both lengths, the three scans: doc_off is complete when this has run
static cudaError_t wf_sizes(const uint8_t* cols, const uint64_t* col_off, const uint64_t* rec_off, const uint8_t* rec_cols, const uint64_t* rec_col_off,
                            const int64_t* created, uint32_t n, uint32_t m, uint64_t* doc_off, uint32_t* summary, uint8_t* state,
                            const WorkflowScratch& S, cudaStream_t st, launch::LaunchLog* lg) {
    cudaError_t e = launch::vcw_records(rec_cols, rec_col_off, created, rec_off, m, S.cls, S.id_off + 1, st, lg);
    if (e == cudaSuccess) e = launch::vcw_sizes(cols, col_off, rec_off, created, S.cls, S.id_off + 1, n, S.msg_off + 1, doc_off + 1, S.arr, summary,
                                                state, st, lg);
    if (e == cudaSuccess) e = launch::offsets_from_lengths(S.msg_off, n, S.scan, st, lg);
    if (e == cudaSuccess) e = launch::offsets_from_lengths(doc_off, n, S.scan, st, lg);
    if (e == cudaSuccess && m) e = launch::offsets_from_lengths(S.id_off, m, S.scan, st, lg);
    return e;
}
// both byte strings, the signatures, the proofValues
static cudaError_t wf_finish(afc_ctx* ctx, const uint8_t* d_exp, uint32_t n_keys, const uint32_t* key_index, const uint8_t* cols, const uint64_t* col_off,
                             const uint64_t* rec_off, const uint8_t* rec_cols, const uint64_t* rec_col_off, const int64_t* created, uint32_t n, uint32_t m,
                             uint8_t* docs, const uint64_t* doc_off, uint8_t* pv, const uint8_t* state, const uint32_t* summary, const WorkflowScratch& S,
                             cudaStream_t st, launch::LaunchLog* lg) {
    cudaError_t e = launch::vcw_fill(cols, col_off, rec_off, created, summary, state, S.arr, n, S.msg_off, S.msgs, doc_off, docs, st, lg);
    if (e == cudaSuccess) e = launch::vcw_ids(rec_cols, rec_col_off, rec_off, n, m, state, S.arr, S.id_off, S.msg_off, S.msgs, doc_off, docs, st, lg);
    if (e == cudaSuccess) e = launch::ed_sign_expanded_batch(ctx->comb, afc_internal_sign_table(ctx), d_exp, n_keys, key_index, S.msgs, S.msg_off, n,
                                                             S.sigs, st, lg);
    if (e == cudaSuccess) e = launch::vcw_proof(S.sigs, state, n, doc_off, docs, pv, st, lg);
    return e;
}
static int wf_check(afc_ctx* ctx, const uint8_t* expanded96, uint32_t n_keys, const uint32_t* key_index, const uint8_t* cols, const uint64_t* col_off,
                    const uint64_t* rec_off, const uint64_t* rec_col_off, uint32_t n, const uint8_t* docs, const uint64_t* doc_off,
                    const uint8_t* proof_values, const uint8_t* state, const uint32_t* summary) {
    if (!ctx || !col_off || !rec_off || !rec_col_off || !doc_off) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    if (!expanded96 || n_keys == 0 || !key_index || !cols || !docs || !proof_values || !state || !summary) return AFC_EINVAL;
    return AFC_OK;
}

int afc_vc_issue_workflow_batch_dev(afc_ctx* ctx, const uint8_t* d_expanded96, uint32_t n_keys, const uint32_t* d_key_index, const uint8_t* d_cols,
                                    const uint64_t* d_col_off, const uint64_t* d_rec_off, const uint8_t* d_rec_cols, const uint64_t* d_rec_col_off,
                                    const int64_t* d_created_at, uint32_t n, uint8_t* d_docs, uint64_t docs_cap, uint64_t* d_doc_off,
                                    uint8_t* d_proof_values, uint8_t* d_state, uint32_t* d_summary, void* stream) {
    int rc = wf_check(ctx, d_expanded96, n_keys, d_key_index, d_cols, d_col_off, d_rec_off, d_rec_col_off, n, d_docs, d_doc_off, d_proof_values,
                      d_state, d_summary);
    if (rc != AFC_OK || n == 0) return rc;
    if (!aligned16(d_expanded96)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    CallLog lc(ctx);
    uint64_t ends[6];                       // the ends of the three offset arrays bound the documents: gathered by one thread, read once
    {
        uint64_t* d_ends = nullptr;
        CK(cudaMallocAsync((void**)&d_ends, sizeof ends, st));
        cudaError_t e = launch::vcw_ends(d_col_off, d_rec_off, d_rec_col_off, n, d_ends, st, lc);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ends, d_ends, sizeof ends, cudaMemcpyDeviceToHost, st);
        cudaFreeAsync(d_ends, st);
        CK(e);
        CK(cudaStreamSynchronize(st));
    }
    if (ends[1] < ends[0] || ends[3] < ends[2] || ends[5] < ends[4] || ends[3] - ends[2] > 0xffffffffull) return AFC_EINVAL;
    const uint32_t m = (uint32_t)(ends[3] - ends[2]);
    if (m && (!d_rec_cols || !d_created_at)) return AFC_EINVAL;
    const uint64_t bound = wf_doc_bound(n, ends[1] - ends[0], m, ends[5] - ends[4]);
    if (docs_cap < bound) return AFC_EINVAL;
    uint8_t* scratch = nullptr;
    WorkflowScratch S;
    CK(pool_carve(&scratch, st, [&](Carve& k) { wf_scratch(k, S, n, m, bound); }));
    cudaError_t e = wf_sizes(d_cols, d_col_off, d_rec_off, d_rec_cols, d_rec_col_off, d_created_at, n, m, d_doc_off, d_summary, d_state, S, st, lc);
    if (e == cudaSuccess) e = wf_finish(ctx, d_expanded96, n_keys, d_key_index, d_cols, d_col_off, d_rec_off, d_rec_cols, d_rec_col_off, d_created_at, n, m,
                                        d_docs, d_doc_off, d_proof_values, d_state, d_summary, S, st, lc);
    cudaFreeAsync(scratch, st);
    CK(e);
    return AFC_OK;
}

int afc_vc_issue_workflow_batch(afc_ctx* ctx, const uint8_t* expanded96, uint32_t n_keys, const uint32_t* key_index, const uint8_t* cols,
                                const uint64_t* col_off, const uint64_t* rec_off, const uint8_t* rec_cols, const uint64_t* rec_col_off,
                                const int64_t* created_at, uint32_t n, uint8_t* docs, uint64_t docs_cap, uint64_t* doc_off, uint8_t* proof_values,
                                uint8_t* state, uint32_t* summary) {
    int rc = wf_check(ctx, expanded96, n_keys, key_index, cols, col_off, rec_off, rec_col_off, n, docs, doc_off, proof_values, state, summary);
    if (rc != AFC_OK) return rc;
    if (n == 0) { doc_off[0] = 0; return AFC_OK; }
    for (uint32_t i = 0; i < n; i++) if (key_index[i] >= n_keys) return AFC_EINVAL;
    uint64_t bad = 0;
    for (size_t k = 0; k < (size_t)n * AFC_WORKFLOW_COLUMNS; k++) bad |= (uint64_t)(col_off[k + 1] < col_off[k]);
    for (uint32_t i = 0; i < n; i++) bad |= (uint64_t)(rec_off[i + 1] < rec_off[i]) | (uint64_t)(rec_off[i + 1] - rec_off[i] > 0xffffffffull);
    if (bad) return AFC_EINVAL;
    for (uint64_t k = 2 * rec_off[0]; k < 2 * rec_off[n]; k++) bad |= (uint64_t)(rec_col_off[k + 1] < rec_col_off[k]);
    if (bad || docs_cap < afc_vc_workflow_bound(col_off, rec_off, rec_col_off, n)) return AFC_EINVAL;
    if (rec_off[n] != rec_off[0] && (!rec_cols || !created_at)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    // Chunks of whole workflows through the ring, as for execution credentials.  A chunk's records travel with it (the kernels index them
    // by absolute record, so the staged record arrays are addressed from a shifted base); a workflow larger than a chunk's byte budget
    // goes alone.
    const uint32_t C = AFC_WORKFLOW_COLUMNS;
    auto measure = [&](uint32_t i0, uint32_t i) {
        const uint64_t r0 = rec_off[i0], r = rec_off[i + 1];
        return (col_off[(size_t)(i + 1) * C] - col_off[(size_t)i0 * C]) + (rec_col_off[2 * r] - rec_col_off[2 * r0]) + 32 * (r - r0);
    };
    uint64_t base = 0;
    return with_device_keys(ctx, expanded96, n_keys, [&](const uint8_t* d_keys) {
        Ring ring(ctx);
        return ring.walk(n, measure, [&](Ring& r) {
            const uint32_t i0 = r.i0, cnt = r.cnt;
            const uint64_t cbase = col_off[(size_t)i0 * C], cbytes = col_off[(size_t)(i0 + cnt) * C] - cbase;
            const uint64_t r0 = rec_off[i0], rbase = rec_col_off[2 * r0], rbytes = rec_col_off[2 * rec_off[i0 + cnt]] - rbase;
            const uint32_t m = (uint32_t)(rec_off[i0 + cnt] - r0);
            const uint64_t dbound = wf_doc_bound(cnt, cbytes, m, rbytes);
            const uint8_t *d_cols, *d_rcols;
            const uint64_t *d_coff, *d_roff, *d_rcoff;
            const uint32_t* d_ki;
            const int64_t* d_cr;
            uint8_t *d_docs, *d_pv, *d_st;
            uint64_t* d_doff;
            uint32_t* d_sum;
            WorkflowScratch S;
            RC(r.stage([&](Stager& k) {
                d_cols = k.in_at(cols, cbase, cbytes, 16);
                d_coff = k.in(col_off, (size_t)i0 * C, (size_t)cnt * C + 1);
                d_ki = k.in(key_index, i0, cnt);
                d_roff = k.in(rec_off, i0, (size_t)cnt + 1);
                d_rcols = k.in_at(rec_cols, rbase, rbytes, 16);
                d_rcoff = k.in(rec_col_off, 2 * r0, m ? 2 * (size_t)m + 1 : 0);
                d_cr = k.in(created_at, 2 * r0, 2 * (size_t)m);
                d_docs = k.take(dbound + 64);
                d_doff = k.take<uint64_t>((size_t)cnt + 1);
                d_pv = k.take((size_t)cnt * 86);
                d_st = k.take(cnt);
                d_sum = k.take<uint32_t>((size_t)cnt * 4);
                wf_scratch(k, S, cnt, m, dbound);
            }));
            d_rcoff -= 2 * r0;                      // absolute record indices stay valid
            d_cr -= 2 * r0;
            CK(wf_sizes(d_cols, d_coff, d_roff, d_rcols, d_rcoff, d_cr, cnt, m, d_doff, d_sum, d_st, S, r.st, r.lc));
            uint64_t bytes;
            RC(r.read(&bytes, {d_doff + cnt}));
            CK(wf_finish(ctx, d_keys, n_keys, d_ki, d_cols, d_coff, d_roff, d_rcols, d_rcoff, d_cr, cnt, m, d_docs, d_doff, d_pv, d_st, d_sum, S, r.st,
                         r.lc));
            RC(r.copy_back({offsets_out(doc_off, i0, d_doff, (size_t)cnt + 1, base), {proof_values, (size_t)i0 * 86, d_pv, (size_t)cnt * 86},
                            {state, i0, d_st, cnt}, {summary, (size_t)i0 * 16, d_sum, (size_t)cnt * 16}, {docs, base, d_docs, bytes}}));
            base += bytes;
            return AFC_OK;
        });
    });
}

// ---------------------------------------------------------------------------------- webhook deliveries
// Bound from the byte counts alone: each delivery's constant text plus at most 6 bytes per column and result byte (a byte escaped as
// backslash-u 00XX or fffd; a number token grows at most 21 / 4 times, 1e20 -> 100000000000000000000).
static uint64_t wh_bound(uint32_t n, uint64_t bytes) { return (uint64_t)n * launch::wh_fixed_bytes() + 6 * bytes; }

uint64_t afc_webhook_bound(const uint64_t* col_off, const uint64_t* result_off, uint32_t n) {
    if (!col_off || !result_off || n == 0) return 0;
    const uint64_t a = col_off[0], b = col_off[(size_t)n * AFC_WEBHOOK_COLUMNS], c = result_off[0], d = result_off[n];
    return wh_bound(n, (b >= a ? b - a : 0) + (d >= c ? d - c : 0));
}

// per-call device scratch: the result tapes, the plans, the HMACs, scan tiles
struct WebhookScratch { uint32_t* tape; uint8_t* plan; uint8_t* mac; uint64_t* scan; };
static void wh_scratch(Carve& k, WebhookScratch& s, uint32_t n, uint64_t result_bytes) {
    s.tape = k.take<uint32_t>(result_bytes / 2 + 1);
    s.plan = k.take(n);
    s.mac = k.take((size_t)n * 32);
    s.scan = (uint64_t*)k.take(launch::json_scan_scratch_bytes(n));
}
static cudaError_t wh_enqueue(const uint8_t* cols, const uint64_t* col_off, const int64_t* dur, const uint8_t* flags, const uint8_t* res,
                              const uint64_t* res_off, const uint8_t* sec, const uint32_t* sec_off, uint32_t n, uint8_t* bodies, uint64_t* body_off,
                              uint8_t* headers, uint8_t* status, const WebhookScratch& S, cudaStream_t st, launch::LaunchLog* lg) {
    cudaError_t e = launch::wh_sizes(cols, col_off, dur, flags, res, res_off, n, S.tape, S.plan, body_off + 1, status, st, lg);
    if (e == cudaSuccess) e = launch::offsets_from_lengths(body_off, n, S.scan, st, lg);
    if (e == cudaSuccess) e = launch::wh_emit(cols, col_off, dur, flags, res, res_off, n, S.tape, S.plan, body_off, bodies, st, lg);
    if (e == cudaSuccess) e = launch::wh_sign(sec, sec_off, flags, status, bodies, body_off, n, S.mac, headers, st, lg);
    return e;
}
static int wh_check(afc_ctx* ctx, const uint8_t* cols, const uint64_t* col_off, const int64_t* dur, const uint8_t* flags, const uint8_t* res,
                    const uint64_t* res_off, const uint8_t* sec, const uint32_t* sec_off, uint32_t n, const uint8_t* bodies, const uint64_t* body_off,
                    const uint8_t* headers, const uint8_t* status) {
    if (!ctx || !col_off || !res_off || !sec_off || !body_off) return AFC_EINVAL;
    if (n && (!cols || !dur || !flags || !bodies || !headers || !status)) return AFC_EINVAL;
    return AFC_OK;
}

int afc_webhook_sign_batch_dev(afc_ctx* ctx, const uint8_t* d_cols, const uint64_t* d_col_off, const int64_t* d_duration_ms, const uint8_t* d_flags,
                               const uint8_t* d_results, const uint64_t* d_result_off, const uint8_t* d_secrets, const uint32_t* d_secret_off,
                               uint32_t n, uint8_t* d_bodies, uint64_t bodies_cap, uint64_t* d_body_off, uint8_t* d_headers, uint8_t* d_status,
                               void* stream) {
    int rc = wh_check(ctx, d_cols, d_col_off, d_duration_ms, d_flags, d_results, d_result_off, d_secrets, d_secret_off, n, d_bodies, d_body_off,
                      d_headers, d_status);
    if (rc != AFC_OK || n == 0) return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    uint64_t ends[4];                       // the column and result bytes bound the bodies and size the tapes: one synchronisation
    CK(cudaMemcpyAsync(&ends[0], d_col_off, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&ends[1], d_col_off + (size_t)n * AFC_WEBHOOK_COLUMNS, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&ends[2], d_result_off, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&ends[3], d_result_off + n, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (ends[1] < ends[0] || ends[3] < ends[2] || bodies_cap < wh_bound(n, (ends[1] - ends[0]) + (ends[3] - ends[2]))) return AFC_EINVAL;
    if ((!d_results && ends[3] != ends[2]) || !d_secrets) return AFC_EINVAL;
    const uint64_t rb = ends[3] - ends[2];
    CallLog lc(ctx);
    uint8_t* scratch = nullptr;
    WebhookScratch S;
    CK(pool_carve(&scratch, st, [&](Carve& k) { wh_scratch(k, S, n, rb); }));
    cudaError_t e = wh_enqueue(d_cols, d_col_off, d_duration_ms, d_flags, d_results, d_result_off, d_secrets, d_secret_off, n, d_bodies, d_body_off,
                               d_headers, d_status, S, st, lc);
    cudaFreeAsync(scratch, st);
    CK(e);
    return AFC_OK;
}

int afc_webhook_sign_batch(afc_ctx* ctx, const uint8_t* cols, const uint64_t* col_off, const int64_t* duration_ms, const uint8_t* flags,
                           const uint8_t* results, const uint64_t* result_off, const uint8_t* secrets, const uint32_t* secret_off, uint32_t n,
                           uint8_t* bodies, uint64_t bodies_cap, uint64_t* body_off, uint8_t* headers, uint8_t* status) {
    int rc = wh_check(ctx, cols, col_off, duration_ms, flags, results, result_off, secrets, secret_off, n, bodies, body_off, headers, status);
    if (rc != AFC_OK) return rc;
    if (n == 0) { body_off[0] = 0; return AFC_OK; }
    uint64_t bad = 0;
    for (size_t k = 0; k < (size_t)n * AFC_WEBHOOK_COLUMNS; k++) bad |= (uint64_t)(col_off[k + 1] < col_off[k]);
    for (uint32_t i = 0; i < n; i++) {
        bad |= (uint64_t)(result_off[i + 1] < result_off[i]) | (uint64_t)(secret_off[i + 1] < secret_off[i]);
        bad |= (uint64_t)(flags[i] & ~(uint32_t)(AFC_WEBHOOK_HAS_DURATION | AFC_WEBHOOK_HAS_ERROR_MESSAGE | AFC_WEBHOOK_HAS_SECRET));
    }
    if (bad || bodies_cap < afc_webhook_bound(col_off, result_off, n)) return AFC_EINVAL;
    if ((!results && result_off[n] != result_off[0]) || (!secrets && secret_off[n] != secret_off[0])) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    // Chunks of deliveries through the ring, as for execution credentials: a chunk's stream is synchronised once after the sizes pass to
    // learn where its bodies end.  The staged secrets are marked secret.
    const uint32_t C = AFC_WEBHOOK_COLUMNS;
    auto measure = [&](uint32_t i0, uint32_t i) {
        return (col_off[(size_t)(i + 1) * C] - col_off[(size_t)i0 * C]) + (result_off[i + 1] - result_off[i0]);
    };
    uint64_t base = 0;
    Ring ring(ctx);
    return ring.walk(n, measure, [&](Ring& r) {
        const uint32_t i0 = r.i0, cnt = r.cnt;
        const uint64_t cbase = col_off[(size_t)i0 * C], cbytes = col_off[(size_t)(i0 + cnt) * C] - cbase;
        const uint64_t rbase = result_off[i0], rbytes = result_off[i0 + cnt] - rbase;
        const uint8_t *d_cols, *d_fl, *d_res, *d_sec;
        const uint64_t *d_coff, *d_roff;
        const uint32_t* d_soff;
        const int64_t* d_dur;
        uint8_t *d_bodies, *d_h, *d_st;
        uint64_t* d_boff;
        WebhookScratch S;
        RC(r.stage([&](Stager& k) {
            d_cols = k.in_at(cols, cbase, cbytes, 16);
            d_coff = k.in(col_off, (size_t)i0 * C, (size_t)cnt * C + 1);
            d_dur = k.in(duration_ms, i0, cnt);
            d_fl = k.in(flags, i0, cnt);
            d_res = k.in_at(results, rbase, rbytes, 16);
            d_roff = k.in(result_off, i0, (size_t)cnt + 1);
            d_sec = k.in_at(secrets, secret_off[i0], secret_off[i0 + cnt] - secret_off[i0], 4, true);
            d_soff = k.in(secret_off, i0, (size_t)cnt + 1);
            d_bodies = k.take(wh_bound(cnt, cbytes + rbytes) + 64);
            d_boff = k.take<uint64_t>((size_t)cnt + 1);
            d_h = k.take((size_t)cnt * 71);
            d_st = k.take(cnt);
            wh_scratch(k, S, cnt, rbytes);
        }));
        CK(launch::wh_sizes(d_cols, d_coff, d_dur, d_fl, d_res, d_roff, cnt, S.tape, S.plan, d_boff + 1, d_st, r.st, r.lc));
        CK(launch::offsets_from_lengths(d_boff, cnt, S.scan, r.st, r.lc));
        uint64_t bytes;
        RC(r.read(&bytes, {d_boff + cnt}));
        CK(launch::wh_emit(d_cols, d_coff, d_dur, d_fl, d_res, d_roff, cnt, S.tape, S.plan, d_boff, d_bodies, r.st, r.lc));
        CK(launch::wh_sign(d_sec, d_soff, d_fl, d_st, d_bodies, d_boff, cnt, S.mac, d_h, r.st, r.lc));
        RC(r.copy_back({offsets_out(body_off, i0, d_boff, (size_t)cnt + 1, base), {headers, (size_t)i0 * 71, d_h, (size_t)cnt * 71},
                        {status, i0, d_st, cnt}, {bodies, base, d_bodies, bytes}}));
        base += bytes;
        return AFC_OK;
    });
}

// ---------------------------------------------------------------------------------- registering agent DIDs
// Bounds from the three offset arrays' ends alone (afc_didreg.cuh): per request its frame with two 10-digit counts, its agent's identity
// with the longest path and 6 bytes per node-id and server-id byte; per id its map entry with the longest path and type, and 6 bytes per
// id byte for each of its two appearances (the key, function_name).  Empty and shadowed ids write nothing, so the bound only gains there.
static uint64_t didr_bound(uint32_t n, uint64_t node_bytes, uint64_t server_len, uint64_t m, uint64_t id_bytes) {
    return (uint64_t)n * (launch::didr_req_fixed() + 6 * server_len) + 6 * node_bytes + m * launch::didr_per_id_fixed() + 12 * id_bytes;
}

uint64_t afc_did_register_bound(const uint64_t* node_off, const uint64_t* id_idx, const uint64_t* id_off, uint32_t n, uint64_t server_id_len) {
    if (!node_off || !id_idx || !id_off || n == 0) return 0;
    const uint64_t a = node_off[0], b = node_off[n], r0 = id_idx[0], r1 = id_idx[2 * (size_t)n];
    const uint64_t nb = b >= a ? b - a : 0;
    if (r1 < r0) return didr_bound(n, nb, server_id_len, 0, 0);
    const uint64_t c = id_off[r0], d = id_off[r1];
    return didr_bound(n, nb, server_id_len, r1 - r0, d >= c ? d - c : 0);
}

// per-call device scratch (launch::DidrArgs); the derived seeds are secret
static void didr_scratch(Carve& k, launch::DidrArgs& A, uint32_t n, uint32_t m) {
    A.list = k.take<uint32_t>(m);
    A.flags = k.take(m);
    A.esc = k.take<uint64_t>(m);
    A.nz = k.take<uint64_t>((size_t)m + 1);
    A.rank = k.take<uint32_t>(m);
    A.before = k.take<uint64_t>(m);
    A.map_bytes = k.take<uint64_t>((size_t)n * 2);
    A.map_cnt = k.take<uint32_t>((size_t)n * 2);
    A.seeds = k.take(((size_t)n + m) * 32, true);
    A.scan = (uint64_t*)k.take(launch::json_scan_scratch_bytes(n > m ? n : m));
}

int afc_did_register_batch_dev(afc_ctx* ctx, const uint8_t* d_master_seed, const uint8_t* server_id, uint64_t server_id_len, const uint8_t* d_node_ids,
                               const uint64_t* d_node_off, const uint32_t* d_agent_index, const uint64_t* d_id_idx, const uint8_t* d_ids,
                               const uint64_t* d_id_off, uint32_t n, uint64_t* d_comp_off, uint8_t* d_expanded96, uint8_t* d_pks, uint8_t* d_dids,
                               uint8_t* d_paths, uint8_t* d_comp_flags, uint8_t* d_body, uint64_t body_cap, uint64_t* d_body_off, void* stream) {
    if (!ctx || !d_node_off || !d_id_idx || !d_id_off || !d_comp_off || !d_body_off) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    if (!d_master_seed || !d_node_ids || !d_agent_index || !d_expanded96 || !d_pks || !d_dids || !d_paths || !d_comp_flags || !d_body ||
        (server_id_len && !server_id))
        return AFC_EINVAL;
    if (!aligned16(d_master_seed) || !aligned16(d_expanded96) || !aligned16(d_pks) || !aligned16(d_paths)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    CallLog lc(ctx);
    uint64_t ends[6];                       // the ends of the three offset arrays bound the bodies: gathered by one thread, read once
    {
        uint64_t* d_ends = nullptr;
        CK(cudaMallocAsync((void**)&d_ends, sizeof ends, st));
        cudaError_t e = launch::didr_ends(d_node_off, d_id_idx, d_id_off, n, d_ends, st, lc);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ends, d_ends, sizeof ends, cudaMemcpyDeviceToHost, st);
        cudaFreeAsync(d_ends, st);
        CK(e);
        CK(cudaStreamSynchronize(st));
    }
    if (ends[1] < ends[0] || ends[3] < ends[2] || ends[5] < ends[4] || ends[3] - ends[2] + n > 0xffffffffull) return AFC_EINVAL;
    const uint32_t m = (uint32_t)(ends[3] - ends[2]);
    if (ends[5] > ends[4] && !d_ids) return AFC_EINVAL;
    if (body_cap < didr_bound(n, ends[1] - ends[0], server_id_len, m, ends[5] - ends[4])) return AFC_EINVAL;
    uint8_t* scratch = nullptr;
    launch::DidrArgs A{};
    uint8_t* d_server;
    CK(pool_carve(&scratch, st, [&](Carve& k) {
        didr_scratch(k, A, n, m);
        d_server = k.take(server_id_len + 16);
    }));
    A.comb = ctx->comb; A.ct16 = afc_internal_sign_table(ctx);
    A.master = d_master_seed; A.h = did_hash(server_id, server_id_len) & 0x7fffffffu; A.server = d_server; A.server_len = server_id_len;
    A.nodes = d_node_ids; A.node_off = d_node_off; A.agent_index = d_agent_index; A.id_idx = d_id_idx; A.ids = d_ids; A.id_off = d_id_off;
    A.n = n; A.m = m;
    A.comp_off = d_comp_off; A.expanded96 = d_expanded96; A.pks = d_pks; A.dids = d_dids; A.paths = d_paths; A.comp_flags = d_comp_flags;
    A.body = d_body; A.body_off = d_body_off;
    cudaError_t e = server_id_len ? cudaMemcpyAsync(d_server, server_id, server_id_len, cudaMemcpyHostToDevice, st) : cudaSuccess;
    if (e == cudaSuccess) e = launch::didr_register(A, st, lc);
    const cudaError_t wipe = cudaMemsetAsync(A.seeds, 0, ((size_t)n + m) * 32, st);       // derived seeds do not outlive the call
    cudaFreeAsync(scratch, st);
    CK(e);
    CK(wipe);
    return AFC_OK;
}

// Device bytes one chunk stages (its arena, to within alignment): inputs, per component its outputs (96 + 32 + 55 + 48 + 1) and seed, per id
// its scratch, and the body bound.  kChunkBytes caps this; a request over it goes alone.
static uint64_t didr_chunk_bytes(uint32_t cnt, uint64_t nbytes, uint64_t server_len, uint64_t mc, uint64_t ibytes) {
    return nbytes + ibytes + 64 * (uint64_t)cnt + 48 * mc + 264 * ((uint64_t)cnt + mc) + didr_bound(cnt, nbytes, server_len, mc, ibytes);
}

// The host-buffer call: chunks of whole requests through one slot of the ring, one after another (the expansion dominates, so there is
// little copy time to overlap).  A chunk's ids travel with it: the kernels index them by absolute id, so the staged arrays are addressed
// from a shifted base.  A request larger than a chunk's byte budget goes alone.  The master seed, the derived seeds, the expanded keys and
// the bodies (every private JWK) are secret.
int afc_did_register_batch(afc_ctx* ctx, const uint8_t* master_seed, const uint8_t* server_id, uint64_t server_id_len, const uint8_t* node_ids,
                           const uint64_t* node_off, const uint32_t* agent_index, const uint64_t* id_idx, const uint8_t* ids, const uint64_t* id_off,
                           uint32_t n, uint64_t* comp_off, uint8_t* expanded96, uint8_t* pks, uint8_t* dids, uint8_t* paths, uint8_t* comp_flags,
                           uint8_t* body, uint64_t body_cap, uint64_t* body_off) {
    if (!ctx || !node_off || !id_idx || !id_off || !comp_off || !body_off) return AFC_EINVAL;
    if (n == 0) { comp_off[0] = 0; body_off[0] = 0; return AFC_OK; }
    if (!master_seed || !node_ids || !agent_index || !expanded96 || !pks || !dids || !paths || !comp_flags || !body || (server_id_len && !server_id))
        return AFC_EINVAL;
    if (!monotone(node_off, n) || !monotone(id_idx, 2 * n)) return AFC_EINVAL;
    const uint64_t r_first = id_idx[0], r_last = id_idx[2 * (size_t)n];
    if (r_last - r_first + n > 0xffffffffull) return AFC_EINVAL;
    uint64_t bad = 0;
    for (uint64_t k = r_first; k < r_last; k++) bad |= (uint64_t)(id_off[k + 1] < id_off[k]);
    if (bad || (id_off[r_last] > id_off[r_first] && !ids)) return AFC_EINVAL;
    if (body_cap < afc_did_register_bound(node_off, id_idx, id_off, n, server_id_len)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    const uint32_t h = did_hash(server_id, server_id_len) & 0x7fffffffu;
    auto measure = [&](uint32_t i0, uint32_t i) {
        const uint64_t r0 = id_idx[2 * (size_t)i0], r = id_idx[2 * (size_t)i + 2];
        return didr_chunk_bytes(i + 1 - i0, node_off[i + 1] - node_off[i0], server_id_len, r - r0, id_off[r] - id_off[r0]);
    };
    uint64_t cbase = 0, bbase = 0;
    {
        Ring ring(ctx, 1);
        RC(ring.walk(n, measure, [&](Ring& r) {
            const uint32_t i0 = r.i0, cnt = r.cnt;
            const uint64_t nb0 = node_off[i0], r0 = id_idx[2 * (size_t)i0], ib0 = id_off[r0], r1 = id_idx[2 * (size_t)(i0 + cnt)];
            const uint32_t mc = (uint32_t)(r1 - r0);
            const size_t slots = (size_t)cnt + mc;
            const uint64_t nbytes = node_off[i0 + cnt] - nb0, ibytes = id_off[r1] - ib0;
            launch::DidrArgs A{};
            RC(r.stage([&](Stager& k) {
                A.nodes = k.in_at(node_ids, nb0, nbytes, 16);
                A.node_off = k.in(node_off, i0, (size_t)cnt + 1);
                A.agent_index = k.in(agent_index, i0, cnt);
                A.id_idx = k.in(id_idx, 2 * (size_t)i0, 2 * (size_t)cnt + 1);
                A.ids = k.in_at(ids, ib0, ibytes, 16);
                A.id_off = k.in(id_off, r0, (size_t)mc + 1);
                A.master = k.in(master_seed, 0, 32, true);
                A.server = k.in(server_id, 0, server_id_len);
                A.comp_off = k.take<uint64_t>((size_t)cnt + 1);
                A.expanded96 = k.take(slots * 96, true);
                A.pks = k.take(slots * 32);
                A.dids = k.take(slots * AFC_DID_CHARS);
                A.paths = k.take(slots * AFC_DID_PATH_SLOT);
                A.comp_flags = k.take(slots);
                A.body = k.take(didr_bound(cnt, nbytes, server_id_len, mc, ibytes) + 64, true);
                A.body_off = k.take<uint64_t>((size_t)cnt + 1);
                didr_scratch(k, A, cnt, mc);
            }));
            A.id_off -= r0;                         // absolute id indices stay valid
            A.comb = ctx->comb; A.ct16 = afc_internal_sign_table(ctx);
            A.h = h; A.server_len = server_id_len;
            A.n = cnt; A.m = mc;
            CK(launch::didr_register(A, r.st, r.lc));
            uint64_t end[2];                        // components, body bytes
            RC(r.read(end, {A.comp_off + cnt, A.body_off + cnt}));
            RC(r.copy_back({offsets_out(comp_off, i0, A.comp_off, (size_t)cnt + 1, cbase), {expanded96, 96 * cbase, A.expanded96, end[0] * 96, true},
                            {pks, 32 * cbase, A.pks, end[0] * 32}, {dids, AFC_DID_CHARS * cbase, A.dids, end[0] * AFC_DID_CHARS},
                            {paths, AFC_DID_PATH_SLOT * cbase, A.paths, end[0] * AFC_DID_PATH_SLOT}, {comp_flags, cbase, A.comp_flags, end[0]},
                            {body, bbase, A.body, end[1], true}, offsets_out(body_off, i0, A.body_off, (size_t)cnt + 1, bbase)}));
            cbase += end[0];
            bbase += end[1];
            return AFC_OK;
        }));
    }
    const size_t tail = (size_t)((uint64_t)n + (r_last - r_first) - cbase);     // the empty ids' entries: zeros, as the _dev call leaves them
    memset(expanded96 + 96 * cbase, 0, tail * 96);
    memset(pks + 32 * cbase, 0, tail * 32);
    memset(dids + AFC_DID_CHARS * cbase, 0, tail * AFC_DID_CHARS);
    memset(paths + AFC_DID_PATH_SLOT * cbase, 0, tail * AFC_DID_PATH_SLOT);
    memset(comp_flags + cbase, 0, tail);
    return AFC_OK;
}

// ---------------------------------------------------------------------------------- re-registering known agents
// Bounds from the five offset arrays' ends alone (afc_didrereg.cuh): per request its frame with the longest message and the agent's stored
// identity, 6 bytes per agent-column and server-id byte; per request id what afc_did_register_bound allows it; per registered component
// its stored entry, 6 bytes per column byte.  Every body lists either the survivors or the new ids, so the bound only gains there.
static uint64_t didrr_bound(uint32_t n, uint64_t agent_bytes, uint64_t server_len, uint64_t m, uint64_t id_bytes, uint64_t G, uint64_t reg_bytes) {
    return (uint64_t)n * (launch::didrr_req_fixed() + 6 * server_len) + 6 * agent_bytes + m * launch::didr_per_id_fixed() + 12 * id_bytes +
           G * launch::didrr_per_reg_fixed() + 6 * reg_bytes;
}

uint64_t afc_did_reregister_bound(const uint64_t* agent_col_off, const uint64_t* id_idx, const uint64_t* id_off, const uint64_t* reg_idx,
                                  const uint64_t* reg_col_off, uint32_t n, uint64_t server_id_len) {
    if (!agent_col_off || !id_idx || !id_off || !reg_idx || !reg_col_off || n == 0) return 0;
    const uint64_t a = agent_col_off[0], b = agent_col_off[3 * (size_t)n];
    const uint64_t r0 = id_idx[0], r1 = id_idx[2 * (size_t)n], g0 = reg_idx[0], g1 = reg_idx[2 * (size_t)n];
    uint64_t m = 0, ib = 0, G = 0, rb = 0;
    if (r1 >= r0) {
        const uint64_t c = id_off[r0], d = id_off[r1];
        m = r1 - r0; ib = d >= c ? d - c : 0;
    }
    if (g1 >= g0) {
        const uint64_t c = reg_col_off[5 * g0], d = reg_col_off[5 * g1];
        G = g1 - g0; rb = d >= c ? d - c : 0;
    }
    return didrr_bound(n, b >= a ? b - a : 0, server_id_len, m, ib, G, rb);
}

// per-call device scratch (launch::DidrrArgs); the derived seeds are secret
static void didrr_scratch(Carve& k, launch::DidrrArgs& A, uint32_t n, uint32_t m, uint32_t G) {
    A.rflags = k.take(G);
    A.ebytes = k.take<uint64_t>(G);
    A.iflags = k.take(m);
    A.esc = k.take<uint64_t>(m);
    A.rank = k.take<uint32_t>((size_t)G + m);
    A.before = k.take<uint64_t>((size_t)G + m);
    A.bad = k.take<uint32_t>(n);
    A.agent_bytes = k.take<uint64_t>(n);
    A.map_bytes = k.take<uint64_t>((size_t)n * 4);
    A.map_cnt = k.take<uint32_t>((size_t)n * 4);
    A.seeds = k.take((size_t)n * 64, true);
    A.scan = (uint64_t*)k.take(launch::json_scan_scratch_bytes(n));
}

int afc_did_reregister_batch_dev(afc_ctx* ctx, const uint8_t* d_master_seed, const uint8_t* server_id, uint64_t server_id_len, const uint8_t* d_agent_cols,
                                 const uint64_t* d_agent_col_off, const uint32_t* d_agent_index, const uint64_t* d_id_idx, const uint8_t* d_ids,
                                 const uint64_t* d_id_off, const uint64_t* d_reg_idx, const uint8_t* d_reg_cols, const uint64_t* d_reg_col_off, uint32_t n,
                                 uint8_t* d_state, uint32_t* d_counts, uint8_t* d_expanded96, uint8_t* d_pks, uint8_t* d_dids, uint8_t* d_paths,
                                 uint8_t* d_reg_flags, uint8_t* d_id_flags, uint8_t* d_body, uint64_t body_cap, uint64_t* d_body_off, void* stream) {
    if (!ctx || !d_agent_col_off || !d_id_idx || !d_id_off || !d_reg_idx || !d_reg_col_off || !d_body_off) return AFC_EINVAL;
    if (n == 0) return AFC_OK;
    if (!d_master_seed || !d_agent_cols || !d_agent_index || !d_state || !d_counts || !d_expanded96 || !d_pks || !d_dids || !d_paths || !d_body ||
        (server_id_len && !server_id))
        return AFC_EINVAL;
    if (!aligned16(d_master_seed) || !aligned16(d_expanded96) || !aligned16(d_pks) || !aligned16(d_paths)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = (cudaStream_t)stream;
    CallLog lc(ctx);
    uint64_t ends[10];                      // the ends of the five offset arrays bound the bodies: gathered by one thread, read once
    {
        uint64_t* d_ends = nullptr;
        CK(cudaMallocAsync((void**)&d_ends, sizeof ends, st));
        cudaError_t e = launch::didrr_ends(d_agent_col_off, d_id_idx, d_id_off, d_reg_idx, d_reg_col_off, n, d_ends, st, lc);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ends, d_ends, sizeof ends, cudaMemcpyDeviceToHost, st);
        cudaFreeAsync(d_ends, st);
        CK(e);
        CK(cudaStreamSynchronize(st));
    }
    for (int k = 0; k < 10; k += 2)
        if (ends[k + 1] < ends[k]) return AFC_EINVAL;
    if ((ends[3] - ends[2]) + (ends[7] - ends[6]) + 2 * (uint64_t)n > 0xffffffffull) return AFC_EINVAL;
    const uint32_t m = (uint32_t)(ends[3] - ends[2]), G = (uint32_t)(ends[7] - ends[6]);
    if ((ends[5] > ends[4] && !d_ids) || (ends[9] > ends[8] && !d_reg_cols) || (m && !d_id_flags) || (G && !d_reg_flags)) return AFC_EINVAL;
    if (body_cap < didrr_bound(n, ends[1] - ends[0], server_id_len, m, ends[5] - ends[4], G, ends[9] - ends[8])) return AFC_EINVAL;
    uint8_t* scratch = nullptr;
    launch::DidrrArgs A{};
    uint8_t* d_server;
    CK(pool_carve(&scratch, st, [&](Carve& k) {
        didrr_scratch(k, A, n, m, G);
        d_server = k.take(server_id_len + 16);
    }));
    A.comb = ctx->comb; A.ct16 = afc_internal_sign_table(ctx);
    A.master = d_master_seed; A.h = did_hash(server_id, server_id_len) & 0x7fffffffu; A.server = d_server; A.server_len = server_id_len;
    A.agent_cols = d_agent_cols; A.agent_col_off = d_agent_col_off; A.agent_index = d_agent_index;
    A.id_idx = d_id_idx; A.ids = d_ids; A.id_off = d_id_off; A.reg_idx = d_reg_idx; A.reg_cols = d_reg_cols; A.reg_col_off = d_reg_col_off;
    A.n = n; A.m = m; A.G = G;
    A.state = d_state; A.counts = d_counts; A.expanded96 = d_expanded96; A.pks = d_pks; A.dids = d_dids; A.paths = d_paths;
    A.reg_flags = d_reg_flags; A.id_flags = d_id_flags; A.body = d_body; A.body_off = d_body_off;
    cudaError_t e = server_id_len ? cudaMemcpyAsync(d_server, server_id, server_id_len, cudaMemcpyHostToDevice, st) : cudaSuccess;
    if (e == cudaSuccess) e = launch::didrr_reregister(A, st, lc);
    const cudaError_t wipe = cudaMemsetAsync(A.seeds, 0, (size_t)n * 64, st);             // derived seeds do not outlive the call
    cudaFreeAsync(scratch, st);
    CK(e);
    CK(wipe);
    return AFC_OK;
}

// Device bytes one chunk stages (its arena, to within alignment): inputs and their offsets, per request its outputs and two key slots
// (2 x (96 + 32 + 55 + 48) + a seed each) and scratch, per id and component its flags and scratch, and the body bound.  kChunkBytes caps
// this; a request over it goes alone.
static uint64_t didrr_chunk_bytes(uint32_t cnt, uint64_t abytes, uint64_t server_len, uint64_t mc, uint64_t ibytes, uint64_t gc, uint64_t rbytes) {
    return abytes + ibytes + rbytes + 8 * (8 * (uint64_t)cnt + mc + 5 * gc) + 640 * (uint64_t)cnt + 32 * (mc + gc) +
           didrr_bound(cnt, abytes, server_len, mc, ibytes, gc, rbytes);
}

// The host-buffer call: chunks of whole requests through one slot of the ring, one after another, as afc_did_register_batch runs.  The
// kernels index ids and components by absolute index, so their staged arrays are addressed from shifted bases.  The master seed, the
// derived seeds, the expanded keys and the bodies (the private JWKs of new components) are secret.
int afc_did_reregister_batch(afc_ctx* ctx, const uint8_t* master_seed, const uint8_t* server_id, uint64_t server_id_len, const uint8_t* agent_cols,
                             const uint64_t* agent_col_off, const uint32_t* agent_index, const uint64_t* id_idx, const uint8_t* ids, const uint64_t* id_off,
                             const uint64_t* reg_idx, const uint8_t* reg_cols, const uint64_t* reg_col_off, uint32_t n, uint8_t* state, uint32_t* counts,
                             uint8_t* expanded96, uint8_t* pks, uint8_t* dids, uint8_t* paths, uint8_t* reg_flags, uint8_t* id_flags, uint8_t* body,
                             uint64_t body_cap, uint64_t* body_off) {
    if (!ctx || !agent_col_off || !id_idx || !id_off || !reg_idx || !reg_col_off || !body_off) return AFC_EINVAL;
    if (n == 0) { body_off[0] = 0; return AFC_OK; }
    if (!master_seed || !agent_cols || !agent_index || !state || !counts || !expanded96 || !pks || !dids || !paths || !body ||
        (server_id_len && !server_id))
        return AFC_EINVAL;
    if (!monotone(agent_col_off, 3 * n) || !monotone(id_idx, 2 * n) || !monotone(reg_idx, 2 * n)) return AFC_EINVAL;
    const uint64_t r_first = id_idx[0], r_last = id_idx[2 * (size_t)n], g_first = reg_idx[0], g_last = reg_idx[2 * (size_t)n];
    if ((r_last - r_first) + (g_last - g_first) + 2 * (uint64_t)n > 0xffffffffull) return AFC_EINVAL;
    uint64_t bad = 0;
    for (uint64_t k = r_first; k < r_last; k++) bad |= (uint64_t)(id_off[k + 1] < id_off[k]);
    for (uint64_t k = 5 * g_first; k < 5 * g_last; k++) bad |= (uint64_t)(reg_col_off[k + 1] < reg_col_off[k]);
    if (bad || (id_off[r_last] > id_off[r_first] && !ids) || (reg_col_off[5 * g_last] > reg_col_off[5 * g_first] && !reg_cols) ||
        (r_last > r_first && !id_flags) || (g_last > g_first && !reg_flags))
        return AFC_EINVAL;
    if (body_cap < afc_did_reregister_bound(agent_col_off, id_idx, id_off, reg_idx, reg_col_off, n, server_id_len)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    const uint32_t h = did_hash(server_id, server_id_len) & 0x7fffffffu;
    auto measure = [&](uint32_t i0, uint32_t i) {
        const uint64_t r0 = id_idx[2 * (size_t)i0], r = id_idx[2 * (size_t)i + 2], g0 = reg_idx[2 * (size_t)i0], g = reg_idx[2 * (size_t)i + 2];
        return didrr_chunk_bytes(i + 1 - i0, agent_col_off[3 * (size_t)i + 3] - agent_col_off[3 * (size_t)i0], server_id_len, r - r0, id_off[r] - id_off[r0],
                                 g - g0, reg_col_off[5 * g] - reg_col_off[5 * g0]);
    };
    uint64_t bbase = 0;
    Ring ring(ctx, 1);
    return ring.walk(n, measure, [&](Ring& r) {
        const uint32_t i0 = r.i0, cnt = r.cnt;
        const uint64_t ac0 = agent_col_off[3 * (size_t)i0], abytes = agent_col_off[3 * (size_t)(i0 + cnt)] - ac0;
        const uint64_t r0 = id_idx[2 * (size_t)i0], r1 = id_idx[2 * (size_t)(i0 + cnt)], ib0 = id_off[r0], ibytes = id_off[r1] - ib0;
        const uint64_t g0 = reg_idx[2 * (size_t)i0], g1 = reg_idx[2 * (size_t)(i0 + cnt)], rb0 = reg_col_off[5 * g0], rbytes = reg_col_off[5 * g1] - rb0;
        const uint32_t mc = (uint32_t)(r1 - r0), gc = (uint32_t)(g1 - g0);
        const size_t slots = 2 * (size_t)cnt;
        launch::DidrrArgs A{};
        RC(r.stage([&](Stager& k) {
            A.agent_cols = k.in_at(agent_cols, ac0, abytes, 16);
            A.agent_col_off = k.in(agent_col_off, 3 * (size_t)i0, 3 * (size_t)cnt + 1);
            A.agent_index = k.in(agent_index, i0, cnt);
            A.id_idx = k.in(id_idx, 2 * (size_t)i0, 2 * (size_t)cnt + 1);
            A.ids = k.in_at(ids, ib0, ibytes, 16);
            A.id_off = k.in(id_off, r0, (size_t)mc + 1);
            A.reg_idx = k.in(reg_idx, 2 * (size_t)i0, 2 * (size_t)cnt + 1);
            A.reg_cols = k.in_at(reg_cols, rb0, rbytes, 16);
            A.reg_col_off = k.in(reg_col_off, 5 * g0, 5 * (size_t)gc + 1);
            A.master = k.in(master_seed, 0, 32, true);
            A.server = k.in(server_id, 0, server_id_len);
            A.state = k.take(cnt);
            A.counts = k.take<uint32_t>(4 * (size_t)cnt);
            A.expanded96 = k.take(slots * 96, true);
            A.pks = k.take(slots * 32);
            A.dids = k.take(slots * AFC_DID_CHARS);
            A.paths = k.take(slots * AFC_DID_PATH_SLOT);
            A.reg_flags = k.take(gc);
            A.id_flags = k.take(mc);
            A.body = k.take(didrr_bound(cnt, abytes, server_id_len, mc, ibytes, gc, rbytes) + 64, true);
            A.body_off = k.take<uint64_t>((size_t)cnt + 1);
            didrr_scratch(k, A, cnt, mc, gc);
        }));
        A.id_off -= r0;                             // absolute indices stay valid
        A.reg_col_off -= 5 * g0;
        A.comb = ctx->comb; A.ct16 = afc_internal_sign_table(ctx);
        A.h = h; A.server_len = server_id_len;
        A.n = cnt; A.m = mc; A.G = gc;
        CK(launch::didrr_reregister(A, r.st, r.lc));
        uint64_t bytes;
        RC(r.read(&bytes, {A.body_off + cnt}));
        RC(r.copy_back({{state, i0, A.state, cnt}, {counts, (size_t)i0 * 16, A.counts, (size_t)cnt * 16},
                        {expanded96, 2 * (size_t)i0 * 96, A.expanded96, slots * 96, true}, {pks, 2 * (size_t)i0 * 32, A.pks, slots * 32},
                        {dids, 2 * (size_t)i0 * AFC_DID_CHARS, A.dids, slots * AFC_DID_CHARS},
                        {paths, 2 * (size_t)i0 * AFC_DID_PATH_SLOT, A.paths, slots * AFC_DID_PATH_SLOT},
                        {reg_flags, g0 - g_first, A.reg_flags, gc}, {id_flags, r0 - r_first, A.id_flags, mc},
                        {body, bbase, A.body, bytes, true}, offsets_out(body_off, i0, A.body_off, (size_t)cnt + 1, bbase)}));
        bbase += bytes;
        return AFC_OK;
    });
}

// ---------------------------------------------------------------------------------- Merkle log
int afc_merkle_new(afc_ctx* ctx, afc_merkle** out) {
    if (!ctx || !out) return AFC_EINVAL;
    *out = nullptr;
    CK(cudaSetDevice(ctx->device));
    afc_merkle* m = new (std::nothrow) afc_merkle();
    if (!m) return AFC_ENOMEM;
    m->ctx = ctx;
    cudaError_t e = cudaMalloc((void**)&m->d_frontier, 64 * 32);
    if (e == cudaSuccess) e = cudaMalloc((void**)&m->d_root, 32);
    if (e == cudaSuccess) e = cudaMemset(m->d_frontier, 0, 64 * 32);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);     // the log's own stream is non-blocking: it would not wait for that memset
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&m->ev, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(m->ev, m->stream);
    if (e != cudaSuccess) { set_err(ctx, e, "afc_merkle_new"); afc_merkle_free(m); return AFC_ECUDA; }
    *out = m;
    return AFC_OK;
}
void afc_merkle_free(afc_merkle* m) {
    if (!m) return;
    cudaSetDevice(m->ctx->device);
    if (m->stream) { cudaStreamSynchronize(m->stream); cudaStreamDestroy(m->stream); }
    if (m->ev) cudaEventDestroy(m->ev);
    if (m->d_frontier) cudaFree(m->d_frontier);
    if (m->d_root) cudaFree(m->d_root);
    m->lv[0].release(); m->lv[1].release(); m->leaves.release(); m->off.release();
    delete m;
}

// Level schedule (host decides structure from (size, n) only; every hash runs on the device).
// d_h: n node hashes occupying leaf positions [size, size+n).  May alias m->lv[1] but not m->lv[0].
static int merkle_append_hashes_locked(afc_merkle* m, const uint8_t* d_h, uint32_t n, cudaStream_t st) {
    afc_ctx* ctx = m->ctx;
    if (n == 0) return AFC_OK;
    if (!aligned16(d_h)) return AFC_EINVAL;
    CallLog lc(ctx);
    uint64_t s = m->size, e = m->size + n;
    const uint8_t* cur = d_h;
    int h = 0, pp = 0;
    // d_h aliasing lv[1]: first output must go to lv[0]
    CK(m->lv[0].reserve(((size_t)n / 2 + 2) * 32));
    while (e > s) {
        int left = (int)(s & 1);
        uint64_t s2 = s + left;
        int right = (int)(e & 1);
        uint64_t e2 = e - right;
        uint64_t npairs = (e2 - s2) / 2;
        DevBuf& ob = m->lv[pp];
        CK(ob.reserve(((size_t)npairs + 2) * 32));
        CK(launch::merkle_level(cur, ob.p, npairs, left, right, m->d_frontier, h, st, lc));
        cur = ob.p;
        s = s2 / 2 - left;
        e = e2 / 2;
        pp ^= 1;
        h++;
        if (h > 63) return AFC_ESTATE;
    }
    m->size += n;
    return AFC_OK;
}

int afc_merkle_append_hashes_dev(afc_merkle* m, const uint8_t* d_hashes32, uint32_t n, void* stream) {
    if (!m) return AFC_EINVAL;
    afc_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(m->mu);
    // the log state and level buffers are shared across calls: order this stream after whatever touched them last
    CK(cudaStreamWaitEvent((cudaStream_t)stream, m->ev, 0));
    int rc = merkle_append_hashes_locked(m, d_hashes32, n, (cudaStream_t)stream);
    CK(cudaEventRecord(m->ev, (cudaStream_t)stream));
    return rc;
}
int afc_merkle_append_dev(afc_merkle* m, const uint8_t* d_leaves, const uint64_t* d_leaf_off, uint32_t n, void* stream) {
    if (!m) return AFC_EINVAL;
    afc_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(m->mu);
    if (n == 0) return AFC_OK;
    CallLog lc(ctx);
    CK(cudaStreamWaitEvent((cudaStream_t)stream, m->ev, 0));
    int rc = AFC_ECUDA;
    cudaError_t e = m->lv[1].reserve((size_t)n * 32);
    if (e == cudaSuccess) e = launch::merkle_leaf_hashes(d_leaves, d_leaf_off, n, m->lv[1].p, (cudaStream_t)stream, lc);
    if (e == cudaSuccess) rc = merkle_append_hashes_locked(m, m->lv[1].p, n, (cudaStream_t)stream);
    else set_err(ctx, e, "afc_merkle_append_dev");
    cudaEventRecord(m->ev, (cudaStream_t)stream);      // whatever was enqueued must order the next user of the log, also after a failure
    return rc;
}
int afc_merkle_root_dev(afc_merkle* m, uint8_t* d_root32, void* stream) {
    if (!m || !d_root32) return AFC_EINVAL;
    afc_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(m->mu);
    CallLog lc(ctx);
    if (!aligned16(d_root32)) return AFC_EINVAL;
    CK(cudaStreamWaitEvent((cudaStream_t)stream, m->ev, 0));
    CK(launch::merkle_root(m->d_frontier, m->size, d_root32, (cudaStream_t)stream, lc));
    CK(cudaEventRecord(m->ev, (cudaStream_t)stream));
    return AFC_OK;
}
static int merkle_root_host_locked(afc_merkle* m, uint8_t root32[32], uint64_t* tree_size) {
    afc_ctx* ctx = m->ctx;
    CallLog lc(ctx);
    CK(cudaStreamWaitEvent(m->stream, m->ev, 0));
    CK(launch::merkle_root(m->d_frontier, m->size, m->d_root, m->stream, lc));
    if (root32) CK(cudaMemcpyAsync(root32, m->d_root, 32, cudaMemcpyDeviceToHost, m->stream));
    CK(cudaStreamSynchronize(m->stream));
    if (tree_size) *tree_size = m->size;
    return AFC_OK;
}
int afc_merkle_root(afc_merkle* m, uint8_t root32[32], uint64_t* tree_size) {
    if (!m) return AFC_EINVAL;
    afc_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(m->mu);
    return merkle_root_host_locked(m, root32, tree_size);
}
int afc_merkle_append(afc_merkle* m, const uint8_t* leaves, const uint64_t* leaf_off, uint32_t n, uint8_t root32[32], uint64_t* tree_size) {
    if (!m || !leaf_off) return AFC_EINVAL;
    afc_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(m->mu);
    CK(cudaStreamWaitEvent(m->stream, m->ev, 0));
    if (n) {
        if (!monotone(leaf_off, n)) return AFC_EINVAL;
        uint64_t base = leaf_off[0], bytes = leaf_off[n] - base;
        if (bytes && !leaves) return AFC_EINVAL;
        size_t pad = (size_t)(base & 15);
        CK(m->leaves.reserve(bytes + 32)); CK(m->off.reserve((size_t)(n + 1) * 8)); CK(m->lv[1].reserve((size_t)n * 32));
        if (bytes) CK(cudaMemcpyAsync(m->leaves.p + pad, leaves + base, bytes, cudaMemcpyHostToDevice, m->stream));
        CK(cudaMemcpyAsync(m->off.p, leaf_off, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, m->stream));
        CallLog lc(ctx);
        CK(launch::merkle_leaf_hashes(m->leaves.p + pad - base, (const uint64_t*)m->off.p, n, m->lv[1].p, m->stream, lc));
            int rc = merkle_append_hashes_locked(m, m->lv[1].p, n, m->stream);
        if (rc != AFC_OK) return rc;
    }
    return merkle_root_host_locked(m, root32, tree_size);
}
int afc_merkle_append_hashes(afc_merkle* m, const uint8_t* hashes32, uint32_t n, uint8_t root32[32], uint64_t* tree_size) {
    if (!m || (n && !hashes32)) return AFC_EINVAL;
    afc_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(m->mu);
    CK(cudaStreamWaitEvent(m->stream, m->ev, 0));
    if (n) {
        CK(m->lv[1].reserve((size_t)n * 32));
        CK(cudaMemcpyAsync(m->lv[1].p, hashes32, (size_t)n * 32, cudaMemcpyHostToDevice, m->stream));
        int rc = merkle_append_hashes_locked(m, m->lv[1].p, n, m->stream);
        if (rc != AFC_OK) return rc;
    }
    return merkle_root_host_locked(m, root32, tree_size);
}
int afc_merkle_save(afc_merkle* m, uint8_t* state) {
    if (!m || !state) return AFC_EINVAL;
    afc_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(m->mu);
    CK(cudaStreamWaitEvent(m->stream, m->ev, 0));
    CK(cudaStreamSynchronize(m->stream));
    memcpy(state, &m->size, 8);
    CK(cudaMemcpy(state + 8, m->d_frontier, 64 * 32, cudaMemcpyDeviceToHost));
    for (int h = 0; h < 64; h++) if (!((m->size >> h) & 1)) memset(state + 8 + 32 * h, 0, 32);
    return AFC_OK;
}
int afc_merkle_load(afc_merkle* m, const uint8_t* state) {
    if (!m || !state) return AFC_EINVAL;
    afc_ctx* ctx = m->ctx;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(m->mu);
    CK(cudaStreamWaitEvent(m->stream, m->ev, 0));
    CK(cudaStreamSynchronize(m->stream));
    memcpy(&m->size, state, 8);
    CK(cudaMemcpy(m->d_frontier, state + 8, 64 * 32, cudaMemcpyHostToDevice));
    return AFC_OK;
}


// ---------------------------------------------------------------------------------- materialised tree + audit proofs
static int tree_build_common(afc_ctx* ctx, const uint8_t* src, bool src_is_device, uint64_t n, afc_merkle_tree** out) {
    if (!ctx || !out || (n && !src)) return AFC_EINVAL;
    *out = nullptr;
    CK(cudaSetDevice(ctx->device));
    afc_merkle_tree* t = new (std::nothrow) afc_merkle_tree();
    if (!t) return AFC_ENOMEM;
    t->ctx = ctx; t->n = n;
    CallLog lc(ctx);
    cudaError_t e = cudaSuccess;
    uint64_t cur = n;
    while (e == cudaSuccess) {
        uint8_t* p = nullptr;
        e = cudaMalloc((void**)&p, (size_t)(cur ? cur : 1) * 32);
        if (e != cudaSuccess) break;
        t->levels.push_back(p); t->sizes.push_back(cur);
        size_t h = t->levels.size() - 1;
        if (h == 0) {
            if (n) e = cudaMemcpy(p, src, (size_t)n * 32, src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice);
        } else {
            e = launch::merkle_level_promote(t->levels[h - 1], t->sizes[h - 1], p, 0, lc);
        }
        if (cur <= 1) break;
        cur = (cur + 1) / 2;
    }
    if (e == cudaSuccess) e = cudaMalloc((void**)&t->d_levels, t->levels.size() * sizeof(uint8_t*));
    if (e == cudaSuccess) e = cudaMalloc((void**)&t->d_sizes, t->sizes.size() * 8);
    if (e == cudaSuccess) e = cudaMemcpy(t->d_levels, t->levels.data(), t->levels.size() * sizeof(uint8_t*), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(t->d_sizes, t->sizes.data(), t->sizes.size() * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { set_err(ctx, e, "afc_merkle_tree_build"); afc_merkle_tree_free(t); return e == cudaErrorMemoryAllocation ? AFC_ENOMEM : AFC_ECUDA; }
    *out = t;
    return AFC_OK;
}
int afc_merkle_tree_build(afc_ctx* ctx, const uint8_t* leaf_hashes32, uint64_t n, afc_merkle_tree** out) { return tree_build_common(ctx, leaf_hashes32, false, n, out); }
int afc_merkle_tree_build_dev(afc_ctx* ctx, const uint8_t* d_leaf_hashes32, uint64_t n, afc_merkle_tree** out) { return tree_build_common(ctx, d_leaf_hashes32, true, n, out); }
void afc_merkle_tree_free(afc_merkle_tree* t) {
    if (!t) return;
    cudaSetDevice(t->ctx->device);
    for (uint8_t* p : t->levels) if (p) cudaFree(p);
    if (t->d_levels) cudaFree(t->d_levels);
    if (t->d_sizes) cudaFree(t->d_sizes);
    delete t;
}
int afc_merkle_tree_root(afc_merkle_tree* t, uint8_t root32[32], uint64_t* n_leaves, uint32_t* max_proof_nodes) {
    if (!t) return AFC_EINVAL;
    afc_ctx* ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    if (n_leaves) *n_leaves = t->n;
    if (max_proof_nodes) *max_proof_nodes = (uint32_t)(t->levels.size() > 1 ? t->levels.size() - 1 : 1);
    if (root32) {
        if (t->n == 0) {                                   // MTH({}) = SHA-256("") — computed on the device like everything else
            CallLog lc(ctx);
            uint8_t* d = nullptr;
            CK(cudaMalloc((void**)&d, 32));
            cudaError_t e = launch::merkle_root(d, 0, d, 0, lc);
            if (e == cudaSuccess) e = cudaMemcpy(root32, d, 32, cudaMemcpyDeviceToHost);
            cudaFree(d);
            CK(e);
        } else {
            CK(cudaMemcpy(root32, t->levels.back(), 32, cudaMemcpyDeviceToHost));
        }
    }
    return AFC_OK;
}
int afc_merkle_tree_inclusion_proofs(afc_merkle_tree* t, const uint64_t* indices, uint32_t m, uint8_t* proofs, uint32_t* proof_lens) {
    if (!t || (m && (!indices || !proofs || !proof_lens))) return AFC_EINVAL;
    afc_ctx* ctx = t->ctx;
    if (m == 0) return AFC_OK;
    CK(cudaSetDevice(ctx->device));
    for (uint32_t i = 0; i < m; i++) if (indices[i] >= t->n) return AFC_EINVAL;
    const size_t depth = t->levels.size() > 1 ? t->levels.size() - 1 : 1;
    uint64_t* d_idx = nullptr; uint8_t* d_out = nullptr; uint32_t* d_len = nullptr;
    cudaError_t e = cudaMalloc((void**)&d_idx, (size_t)m * 8);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_out, (size_t)m * depth * 32);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_len, (size_t)m * 4);
    if (e == cudaSuccess) e = cudaMemcpy(d_idx, indices, (size_t)m * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(d_out, 0, (size_t)m * depth * 32);             // slots past a path's length come back as zeros
    if (e == cudaSuccess) {
        CallLog lc(ctx);
        e = launch::merkle_gather_proofs((const uint8_t* const*)t->d_levels, t->d_sizes, (int)t->levels.size(), d_idx, m, d_out, d_len, 0, lc);
    }
    if (e == cudaSuccess) e = cudaMemcpy(proofs, d_out, (size_t)m * depth * 32, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess) e = cudaMemcpy(proof_lens, d_len, (size_t)m * 4, cudaMemcpyDeviceToHost);
    cudaFree(d_idx); cudaFree(d_out); cudaFree(d_len);
    CK(e);
    return AFC_OK;
}
int afc_merkle_verify_inclusion_batch(afc_ctx* ctx, const uint8_t* leaf_hashes32, const uint64_t* indices, uint64_t tree_size,
                                      const uint8_t* proofs, const uint32_t* proof_off, const uint8_t root32[32], uint32_t m, uint8_t* ok) {
    if (!ctx || (m && (!leaf_hashes32 || !indices || !proof_off || !root32 || !ok))) return AFC_EINVAL;
    if (m == 0) return AFC_OK;
    CK(cudaSetDevice(ctx->device));
    const size_t pn = proof_off[m];
    if (pn && !proofs) return AFC_EINVAL;
    uint8_t *d_lh = nullptr, *d_pr = nullptr, *d_root = nullptr, *d_ok = nullptr; uint64_t* d_idx = nullptr; uint32_t* d_po = nullptr;
    cudaError_t e = cudaMalloc((void**)&d_lh, (size_t)m * 32);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_pr, (pn ? pn : 1) * 32);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_root, 32);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_ok, m);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_idx, (size_t)m * 8);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_po, (size_t)(m + 1) * 4);
    if (e == cudaSuccess) e = cudaMemcpy(d_lh, leaf_hashes32, (size_t)m * 32, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && pn) e = cudaMemcpy(d_pr, proofs, pn * 32, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_root, root32, 32, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_idx, indices, (size_t)m * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_po, proof_off, (size_t)(m + 1) * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        CallLog lc(ctx);
        e = launch::merkle_verify_inclusion(d_lh, d_idx, tree_size, d_pr, d_po, d_root, m, d_ok, 0, lc);
    }
    if (e == cudaSuccess) e = cudaMemcpy(ok, d_ok, m, cudaMemcpyDeviceToHost);
    cudaFree(d_lh); cudaFree(d_pr); cudaFree(d_root); cudaFree(d_ok); cudaFree(d_idx); cudaFree(d_po);
    CK(e);
    return AFC_OK;
}

// RFC 6962 §2.1.2 PROOF(first, D[n]) read out of the materialised levels.  Every node of the proof is MTH(D[a:b]) with a
// a multiple of 2^l and b = min(a + 2^l, n): exactly node (level l, index a >> l) of the tree (a lone right node is promoted
// unchanged, which is what the RFC's largest-power-of-two split yields for a ragged right edge).
namespace {
void consistency_nodes(uint64_t m, uint64_t lo, uint64_t hi, bool whole, std::vector<std::pair<int, uint64_t>>& out) {
    const uint64_t n = hi - lo;
    auto node = [&](uint64_t a, uint64_t width_pow2) { int l = 0; while ((1ull << l) < width_pow2) l++; out.emplace_back(l, a >> l); };
    auto pow2_ceil = [](uint64_t w) { uint64_t p = 1; while (p < w) p <<= 1; return p; };
    if (m == n) { if (!whole) node(lo, pow2_ceil(n)); return; }
    uint64_t k = 1; while (k * 2 < n) k *= 2;
    if (m <= k) { consistency_nodes(m, lo, lo + k, whole, out); node(lo + k, k); }
    else { consistency_nodes(m - k, lo + k, hi, false, out); node(lo, k); }
}
}  // namespace
int afc_merkle_tree_consistency_proof(afc_merkle_tree* t, uint64_t first, uint8_t* proof, uint32_t* n_nodes) {
    if (!t || !n_nodes || first == 0 || first > t->n) return AFC_EINVAL;
    afc_ctx* ctx = t->ctx;
    CK(cudaSetDevice(ctx->device));
    std::vector<std::pair<int, uint64_t>> nodes;
    consistency_nodes(first, 0, t->n, true, nodes);
    if (nodes.size() && !proof) return AFC_EINVAL;
    for (size_t i = 0; i < nodes.size(); i++) {
        const int l = nodes[i].first; const uint64_t j = nodes[i].second;
        if (l >= (int)t->levels.size() || j >= t->sizes[l]) return AFC_ESTATE;
        CK(cudaMemcpy(proof + 32 * i, t->levels[l] + 32 * j, 32, cudaMemcpyDeviceToHost));
    }
    *n_nodes = (uint32_t)nodes.size();
    return AFC_OK;
}
int afc_merkle_verify_consistency_batch(afc_ctx* ctx, const uint64_t* first_sizes, const uint8_t* first_roots32, uint64_t second_size,
                                        const uint8_t second_root32[32], const uint8_t* proofs, const uint32_t* proof_off, uint32_t m, uint8_t* ok) {
    if (!ctx || (m && (!first_sizes || !first_roots32 || !second_root32 || !proof_off || !ok))) return AFC_EINVAL;
    if (m == 0) return AFC_OK;
    CK(cudaSetDevice(ctx->device));
    const size_t pn = proof_off[m];
    if (pn && !proofs) return AFC_EINVAL;
    uint8_t *d_fr = nullptr, *d_pr = nullptr, *d_sr = nullptr, *d_ok = nullptr; uint64_t* d_fs = nullptr; uint32_t* d_po = nullptr;
    cudaError_t e = cudaMalloc((void**)&d_fr, (size_t)m * 32);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_pr, (pn ? pn : 1) * 32);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_sr, 32);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_ok, m);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_fs, (size_t)m * 8);
    if (e == cudaSuccess) e = cudaMalloc((void**)&d_po, (size_t)(m + 1) * 4);
    if (e == cudaSuccess) e = cudaMemcpy(d_fr, first_roots32, (size_t)m * 32, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && pn) e = cudaMemcpy(d_pr, proofs, pn * 32, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_sr, second_root32, 32, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_fs, first_sizes, (size_t)m * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_po, proof_off, (size_t)(m + 1) * 4, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        CallLog lc(ctx);
        e = launch::merkle_verify_consistency(d_fs, d_fr, second_size, d_sr, d_pr, d_po, m, d_ok, 0, lc);
    }
    if (e == cudaSuccess) e = cudaMemcpy(ok, d_ok, m, cudaMemcpyDeviceToHost);
    cudaFree(d_fr); cudaFree(d_pr); cudaFree(d_sr); cudaFree(d_ok); cudaFree(d_fs); cudaFree(d_po);
    CK(e);
    return AFC_OK;
}

// ---------------------------------------------------------------------------------- NCCL (dlopen, optional)
namespace {
struct nccl_id_t { char internal[128]; };
typedef int (*fn_get_uid)(nccl_id_t*);
typedef int (*fn_init_rank)(void**, int, nccl_id_t, int);
typedef int (*fn_allgather)(const void*, void*, size_t, int, void*, cudaStream_t);
typedef int (*fn_destroy)(void*);
void* nccl_open() {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);      // reuse the copy torch already loaded, if any
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    return h;
}
}  // namespace

int afc_comm_unique_id(uint8_t id128[128]) {
    void* h = nccl_open();
    if (!h) return AFC_ENCCL;
    fn_get_uid f = (fn_get_uid)dlsym(h, "ncclGetUniqueId");
    if (!f) return AFC_ENCCL;
    nccl_id_t id;
    if (f(&id) != 0) return AFC_ENCCL;
    memcpy(id128, id.internal, 128);
    return AFC_OK;
}
int afc_comm_init(afc_ctx* ctx, int nranks, int rank, const uint8_t id128[128]) {
    if (!ctx || nranks < 1 || rank < 0 || rank >= nranks) return AFC_EINVAL;
    if (ctx->nccl_comm) return AFC_ESTATE;
    CK(cudaSetDevice(ctx->device));
    ctx->nccl_lib = nccl_open();
    if (!ctx->nccl_lib) return AFC_ENCCL;
    fn_init_rank f = (fn_init_rank)dlsym(ctx->nccl_lib, "ncclCommInitRank");
    if (!f) return AFC_ENCCL;
    nccl_id_t id; memcpy(id.internal, id128, 128);
    if (f(&ctx->nccl_comm, nranks, id, rank) != 0) { ctx->nccl_comm = nullptr; return AFC_ENCCL; }
    ctx->nranks = nranks; ctx->rank = rank;
    CK(cudaStreamCreateWithFlags(&ctx->comm_stream, cudaStreamNonBlocking));
    CK(cudaMalloc((void**)&ctx->d_comm_buf, (size_t)(nranks + 1) * 32));
    return AFC_OK;
}
int afc_comm_allgather_roots(afc_ctx* ctx, const uint8_t local_root32[32], uint8_t* all_roots) {
    if (!ctx || !local_root32 || !all_roots) return AFC_EINVAL;
    if (!ctx->nccl_comm) return AFC_ESTATE;
    CK(cudaSetDevice(ctx->device));
    fn_allgather f = (fn_allgather)dlsym(ctx->nccl_lib, "ncclAllGather");
    if (!f) return AFC_ENCCL;
    uint8_t* send = ctx->d_comm_buf + (size_t)ctx->nranks * 32;
    CK(cudaMemcpyAsync(send, local_root32, 32, cudaMemcpyHostToDevice, ctx->comm_stream));
    if (f(send, ctx->d_comm_buf, 32, /*ncclUint8*/ 1, ctx->nccl_comm, ctx->comm_stream) != 0) return AFC_ENCCL;
    CK(cudaMemcpyAsync(all_roots, ctx->d_comm_buf, (size_t)ctx->nranks * 32, cudaMemcpyDeviceToHost, ctx->comm_stream));
    CK(cudaStreamSynchronize(ctx->comm_stream));
    return AFC_OK;
}
int afc_comm_destroy(afc_ctx* ctx) {
    if (!ctx) return AFC_EINVAL;
    if (ctx->nccl_comm) {
        fn_destroy f = (fn_destroy)dlsym(ctx->nccl_lib, "ncclCommDestroy");
        if (f) f(ctx->nccl_comm);
        ctx->nccl_comm = nullptr;
    }
    if (ctx->comm_stream) { cudaStreamDestroy(ctx->comm_stream); ctx->comm_stream = nullptr; }
    if (ctx->d_comm_buf) { cudaFree(ctx->d_comm_buf); ctx->d_comm_buf = nullptr; }
    return AFC_OK;
}


// ---------------------------------------------------------------------------------- per-kernel event profiling
int afc_profile_begin(afc_ctx* ctx, int max_launches) {
    if (!ctx || max_launches <= 0) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    std::lock_guard<std::mutex> g(ctx->mu);
    if (ctx->profile) return AFC_ESTATE;
    size_t old = ctx->prof_recs.size();
    if ((size_t)max_launches > old) {
        ctx->prof_recs.resize(max_launches);
        for (size_t i = old; i < ctx->prof_recs.size(); i++) {
            ctx->prof_recs[i].name = nullptr; ctx->prof_recs[i].done = false;
            if (cudaEventCreate(&ctx->prof_recs[i].e0) != cudaSuccess || cudaEventCreate(&ctx->prof_recs[i].e1) != cudaSuccess) return AFC_ECUDA;
        }
    }
    for (auto& r : ctx->prof_recs) r.done = false;
    __atomic_store_n(&ctx->prof_next, 0, __ATOMIC_RELAXED);
    ctx->profile = true;
    return AFC_OK;
}
// Returns the number of distinct kernel names (entries written to out, at most cap).  Launches beyond the pool given to
// afc_profile_begin were not timed: they are reported in the entry named "(untimed)" (count only) so that a short pool is visible.
int afc_profile_end(afc_ctx* ctx, afc_profile_entry* out, int cap) {
    if (!ctx || (cap > 0 && !out)) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());
    std::lock_guard<std::mutex> g(ctx->mu);
    if (!ctx->profile) return AFC_ESTATE;
    ctx->profile = false;
    int n_out = 0;
    const int claimed = __atomic_load_n(&ctx->prof_next, __ATOMIC_RELAXED);
    const int timed = claimed < (int)ctx->prof_recs.size() ? claimed : (int)ctx->prof_recs.size();
    for (int i = 0; i < timed; i++) {
        launch::LaunchRec& r = ctx->prof_recs[i];
        if (!r.done) continue;
        float ms = 0;
        if (cudaEventElapsedTime(&ms, r.e0, r.e1) != cudaSuccess) { cudaGetLastError(); continue; }
        int k = 0;
        for (; k < n_out; k++) if (strncmp(out[k].name, r.name, sizeof(out[k].name) - 1) == 0) break;
        if (k == n_out) {
            if (n_out >= cap) continue;
            memset(&out[k], 0, sizeof(out[k]));
            strncpy(out[k].name, r.name, sizeof(out[k].name) - 1);
            out[k].min_ms = ms; out[k].max_ms = ms;
            n_out++;
        }
        out[k].count++;
        out[k].total_ms += ms;
        if (ms < out[k].min_ms) out[k].min_ms = ms;
        if (ms > out[k].max_ms) out[k].max_ms = ms;
    }
    if (claimed > timed && n_out < cap) {
        memset(&out[n_out], 0, sizeof(out[n_out]));
        strncpy(out[n_out].name, "(untimed)", sizeof(out[n_out].name) - 1);
        out[n_out].count = (uint32_t)(claimed - timed);
        n_out++;
    }
    return n_out;
}

// ---------------------------------------------------------------------------------- diagnostics
// Counts the occurrences of a byte pattern in every lane's staging memory (device slot buffers and pinned bounce buffers), with every
// lane held so that no call runs meanwhile: what a test uses to check that no secret outlives a host-buffer call.
int afc_staging_find(afc_ctx* ctx, const uint8_t* pattern, uint32_t len, uint64_t* hits) {
    if (!ctx || !pattern || !hits || len == 0 || len > 64) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    {
        std::unique_lock<std::mutex> lk(ctx->mu);
        for (;;) {
            bool idle = true;
            for (int i = 0; i < kLanes; i++) idle = idle && !ctx->lanes[i].busy;
            if (idle) break;
            ctx->cv.wait(lk);
        }
        for (int i = 0; i < kLanes; i++) ctx->lanes[i].busy = true;
    }
    struct Release {
        afc_ctx* ctx;
        ~Release() {
            { std::lock_guard<std::mutex> g(ctx->mu); for (int i = 0; i < kLanes; i++) ctx->lanes[i].busy = false; }
            ctx->cv.notify_all();
        }
    } release{ctx};
    uint64_t count = 0;
    auto scan = [&](const uint8_t* p, size_t n) {
        for (const uint8_t* q = p; n >= len;) {
            const uint8_t* f = (const uint8_t*)memchr(q, pattern[0], n - len + 1);
            if (!f) break;
            if (memcmp(f, pattern, len) == 0) count++;
            n -= (size_t)(f + 1 - q);
            q = f + 1;
        }
    };
    constexpr size_t kPiece = 64u << 20;
    std::vector<uint8_t> host;
    for (int i = 0; i < kLanes; i++) {
        for (int w = 0; w < kSlots; w++) {
            Slot& sl = ctx->lanes[i].slot[w];
            if (sl.stream) CK(cudaStreamSynchronize(sl.stream));
            for (size_t at = 0; at < sl.arena.cap; at += kPiece) {      // pieces overlap by len - 1 bytes, so no match is cut in two
                const size_t n = sl.arena.cap - at < kPiece + len - 1 ? sl.arena.cap - at : kPiece + len - 1;
                host.resize(n);
                CK(cudaMemcpy(host.data(), sl.arena.p + at, n, cudaMemcpyDeviceToHost));
                scan(host.data(), n);
            }
            PinBuf* pin[] = {&sl.h_in, &sl.h_out};
            for (PinBuf* b : pin) if (b->p) scan(b->p, b->cap);
        }
    }
    *hits = count;
    return AFC_OK;
}

int afc_selftest(afc_ctx* ctx, uint32_t iters) {
    if (!ctx) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    uint32_t* d = nullptr;
    CK(cudaMalloc((void**)&d, 4));
    CK(cudaMemset(d, 0, 4));
    CallLog lc(ctx);
    cudaError_t e = launch::ed_selftest(iters, d, 0, lc);
    uint32_t bad = 0;
    if (e == cudaSuccess) e = cudaMemcpy(&bad, d, 4, cudaMemcpyDeviceToHost);
    cudaFree(d);
    CK(e);
    return (int)bad;
}
int afc_microbench(afc_ctx* ctx, int which, uint32_t iters, double* ops_per_s, double* ms_out) {
    if (!ctx || !ops_per_s) return AFC_EINVAL;
    CK(cudaSetDevice(ctx->device));
    uint32_t* d = nullptr;
    CK(cudaMalloc((void**)&d, 4));
    const uint32_t threads = 128;
    const uint32_t blocks = (uint32_t)ctx->prop.multiProcessorCount * 8;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CallLog lc(ctx);
    cudaError_t e = cudaSuccess;
    for (int rep = 0; rep < 2 && e == cudaSuccess; rep++) {      // first pass warms up
        cudaEventRecord(e0, 0);
        if (which == 3 || which == 4) e = launch::microbench_hash(which, iters, blocks, threads, d, 0, lc);
        else e = launch::microbench_fe(which, iters, blocks, threads, d, 0, lc);
        cudaEventRecord(e1, 0);
        if (e == cudaSuccess) e = cudaEventSynchronize(e1);
    }
    float ms = 0;
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(d);
    CK(e);
    double per_thread = (which == 3 || which == 4) ? 1.0 : (which >= 20 ? 1.0 : (which >= 10 ? 16.0 : 2.0));   // fe probes: 2 ops / iteration; pipe probes: 16 instr
    *ops_per_s = (double)blocks * threads * iters * per_thread / (ms * 1e-3);
    if (ms_out) *ms_out = ms;
    return AFC_OK;
}

}  // extern "C"
