// Internal launch API between the C-ABI layer (afcrypto.cu) and the kernel translation units
// (k_hash.cu, k_ed25519.cu).  All pointers are DEVICE pointers; every function only enqueues work on
// `s` and returns cudaGetLastError().  Each launch is counted (and optionally timed) through the LaunchLog.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace afc {
namespace launch {

// Launch accounting + optional per-kernel CUDA-event timing (afc_profile_*): when `profile` is set every kernel
// launch is bracketed by two events on its own stream; afcrypto.cu aggregates them by kernel name after a sync.
struct LaunchRec { const char* name; cudaEvent_t e0, e1; bool done; };
struct LaunchLog {
    unsigned long long n = 0;
    bool profile = false;
    LaunchRec* pool = nullptr;       // the context's pool of event pairs; one is claimed per launch (never more than are used)
    int cap = 0;
    int* next = nullptr;             // shared claim counter (atomic on the host)
    LaunchRec* cur = nullptr;
    cudaEvent_t begin(const char* name, cudaStream_t s) {
        ++n;
        if (!profile) return nullptr;
        const int idx = __atomic_fetch_add(next, 1, __ATOMIC_RELAXED);
        if (idx >= cap) return nullptr;
        cur = &pool[idx];
        cur->name = name; cur->done = false;
        cudaEventRecord(cur->e0, s);
        return cur->e1;
    }
    void end(cudaEvent_t e1, cudaStream_t s) { if (e1) { cudaEventRecord(e1, s); cur->done = true; } }
};
#define AFC_LAUNCH(lg, name, stream, ...)            \
    do {                                             \
        cudaEvent_t _e1 = (lg)->begin(name, stream); \
        __VA_ARGS__;                                 \
        (lg)->end(_e1, stream);                      \
    } while (0)

// ---- k_hash.cu
cudaError_t sha256_batch(const uint8_t* msgs, const uint64_t* off, uint32_t n, uint8_t* out32, cudaStream_t s, LaunchLog* lg);
cudaError_t hmac_sha256_batch(const uint8_t* keys, const uint32_t* koff, const uint8_t* msgs, const uint64_t* off, uint32_t n,
                              uint8_t* out32, cudaStream_t s, LaunchLog* lg);
// streaming SHA-256: 108-byte states (Go MarshalBinary layout) in/out, chunk i into state i, digest where final_flags[i]
cudaError_t sha256_update(uint8_t* states, const uint8_t* chunks, const uint64_t* off, uint32_t n, const uint8_t* final_flags, uint8_t* out32,
                          uint8_t* status, cudaStream_t s, LaunchLog* lg);
cudaError_t merkle_leaf_hashes(const uint8_t* leaves, const uint64_t* off, uint32_t n, uint8_t* out32, cudaStream_t s, LaunchLog* lg);
// One tree level.  in: node array whose element 0 has level-index s_idx; npairs pairs starting at element `first`
// (first = 1 when s_idx was odd and the left orphan in[0] merges with frontier[h]); out[carry..] receives the parents.
//   left_merge  : out[0] = H(frontier[h] || in[0])                         (then pairs go to out[1..])
//   right_orphan: frontier[h] = in[first + 2*npairs]
cudaError_t merkle_level(const uint8_t* in, uint8_t* out, uint64_t npairs, int left_merge, int right_orphan,
                         uint8_t* frontier, int h, cudaStream_t s, LaunchLog* lg);
// root from frontier (bits of `size` say which heights are present); size == 0 -> SHA-256("")
cudaError_t merkle_root(const uint8_t* frontier, uint64_t size, uint8_t* out32, cudaStream_t s, LaunchLog* lg);
cudaError_t merkle_level_promote(const uint8_t* in, uint64_t n_in, uint8_t* out, cudaStream_t s, LaunchLog* lg);
cudaError_t merkle_gather_proofs(const uint8_t* const* levels, const uint64_t* sizes, int n_levels, const uint64_t* indices, uint32_t m,
                                 uint8_t* out, uint32_t* lens, cudaStream_t s, LaunchLog* lg);
cudaError_t merkle_verify_inclusion(const uint8_t* leaf_hashes, const uint64_t* indices, uint64_t tree_size, const uint8_t* proofs,
                                    const uint32_t* proof_off, const uint8_t* root, uint32_t m, uint8_t* ok, cudaStream_t s, LaunchLog* lg);
cudaError_t merkle_verify_consistency(const uint64_t* first_sizes, const uint8_t* first_roots, uint64_t second_size, const uint8_t* second_root,
                                      const uint8_t* proofs, const uint32_t* proof_off, uint32_t m, uint8_t* ok, cudaStream_t s, LaunchLog* lg);
size_t json_scan_scratch_bytes(uint32_t n);
cudaError_t json_fill_sizes(const uint8_t* segs, const uint32_t* seg_off, const uint8_t* kinds, uint32_t F, const uint8_t* fields,
                            const uint64_t* field_off, uint32_t n, uint64_t* out_off, uint64_t* scan_scratch, cudaStream_t s, LaunchLog* lg);
cudaError_t json_fill(const uint8_t* segs, const uint32_t* seg_off, const uint8_t* kinds, uint32_t F, const uint8_t* fields,
                      const uint64_t* field_off, uint32_t n, const uint64_t* out_off, uint8_t* out, cudaStream_t s, LaunchLog* lg);
// n lengths in out_off[1..n] -> n+1 offsets (out_off[0] = 0); scan_scratch: json_scan_scratch_bytes(n)
cudaError_t offsets_from_lengths(uint64_t* out_off, uint32_t n, uint64_t* scan_scratch, cudaStream_t s, LaunchLog* lg);
cudaError_t b64url_encode(const uint8_t* in, uint32_t item, uint32_t n, uint8_t* out, cudaStream_t s, LaunchLog* lg);
cudaError_t hex_encode(const uint8_t* in, uint64_t total, uint8_t* out, cudaStream_t s, LaunchLog* lg);
cudaError_t microbench_hash(int which, uint32_t iters, uint32_t blocks, uint32_t threads, uint32_t* sink, cudaStream_t s, LaunchLog* lg);

// ---- k_vcdoc.cu: stored credential documents (afc_vcdoc.cuh).  schema: a VcSchema on the device (vc_schema_bytes()).
size_t vc_schema_bytes();
int vc_schema_host(int doc_kind, void* out);           // builds the host copy of a schema; -1 for an unknown kind
// status: the verdict so far (VC_VALID = a candidate for verification); len_out[i]: signing-message length (0 unless candidate);
// sigs: n x 64 (16-byte aligned); key_index: n; fields: n x 4 or nullptr
cudaError_t vc_parse(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint8_t* dids, const uint32_t* did_off,
                     const uint32_t* slots, uint32_t slot_mask, uint8_t* status, uint64_t* len_out, uint8_t* sigs, uint32_t* key_index,
                     uint32_t* fields, cudaStream_t s, LaunchLog* lg);
// k_vc_parse plus the audit capture: caps = vc_capture_bytes(n), 16-byte aligned
cudaError_t vc_parse_capture(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint8_t* dids, const uint32_t* did_off,
                             const uint32_t* slots, uint32_t slot_mask, uint8_t* status, uint64_t* len_out, uint8_t* sigs, uint32_t* key_index,
                             uint32_t* caps, cudaStream_t s, LaunchLog* lg);
size_t vc_capture_bytes(uint32_t n);
// issue masks of the captured documents against their records (col_off: 10 per record + 1, nullptr for workflow documents)
cudaError_t vc_crosscheck(int kind, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint32_t* caps, const uint8_t* status,
                          const uint8_t* cols, const uint64_t* col_off, uint32_t* issues, cudaStream_t s, LaunchLog* lg);
cudaError_t vc_emit(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint64_t* msg_off, uint8_t* msgs,
                    cudaStream_t s, LaunchLog* lg);
cudaError_t vc_fold(uint8_t* status, const uint8_t* ok, uint32_t n, cudaStream_t s, LaunchLog* lg);

// ---- k_vcjson.cu: credential documents in any JSON spelling (afc_vcjson.cuh).  schema: a VcjSchema on the device (vcj_schema_bytes()).
size_t vcj_schema_bytes();
int vcj_schema_host(int doc_kind, void* out);          // builds the host copy of a schema; -1 for an unknown kind
// the outputs of vc_parse; len_out[i] = length of the re-marshalled signing message (0 unless candidate)
cudaError_t vcj_parse(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint8_t* dids, const uint32_t* did_off,
                      const uint32_t* slots, uint32_t slot_mask, uint8_t* status, uint64_t* len_out, uint8_t* sigs, uint32_t* key_index,
                      uint32_t* fields, cudaStream_t s, LaunchLog* lg);
cudaError_t vcj_emit(const void* schema, const uint8_t* docs, const uint64_t* doc_off, uint32_t n, const uint64_t* msg_off, uint8_t* msgs,
                     cudaStream_t s, LaunchLog* lg);

// ---- k_vcissue.cu: execution credentials issued on the device (afc_vcissue.cuh).  col_off: 14 absolute offsets per credential + 1;
// hashes: 2 x 43 characters per credential (input, output), nullptr without HashSensitiveData
// payload j of 2n (input i = 2i, output i = 2i + 1) -> hashData characters at hashes + 43 j
cudaError_t vci_hashdata(const uint8_t* payloads, const uint64_t* payload_off, const uint8_t* nil, uint32_t m, uint8_t* hashes, cudaStream_t s,
                         LaunchLog* lg);
// the signing-message and stored-document length of each credential (write them to off + 1 for offsets_from_lengths)
cudaError_t vci_sizes(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* hashes, uint32_t n, uint64_t* msg_len,
                      uint64_t* doc_len, cudaStream_t s, LaunchLog* lg);
// both byte strings of each credential; the stored document's proofValue is a placeholder until vci_proof
cudaError_t vci_fill(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* hashes, uint32_t n, const uint64_t* msg_off,
                     uint8_t* msgs, const uint64_t* doc_off, uint8_t* docs, cudaStream_t s, LaunchLog* lg);
// sigs: n x 64, 16-byte aligned -> 86 characters into each stored document and into proof_values (n x 86)
cudaError_t vci_proof(const uint8_t* sigs, uint32_t n, const uint64_t* doc_off, uint8_t* docs, uint8_t* proof_values, cudaStream_t s, LaunchLog* lg);
uint64_t vci_literal_bytes();          // constant text of both document forms together

// ---- k_webhook.cu: webhook deliveries built and signed on the device (afc_webhook.cuh).  col_off: 8 absolute offsets per delivery + 1;
// result_off: n + 1 absolute offsets; tape: (result_off[n] - result_off[0]) / 2 + 1 entries; plan: n bytes kept between the passes
// each body's length (0 for a WH_HOST delivery; write them to body_off + 1 for offsets_from_lengths) and its status
cudaError_t wh_sizes(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* flags, const uint8_t* results,
                     const uint64_t* result_off, uint32_t n, uint32_t* tape, uint8_t* plan, uint64_t* body_len, uint8_t* status, cudaStream_t s,
                     LaunchLog* lg);
cudaError_t wh_emit(const uint8_t* cols, const uint64_t* col_off, const int64_t* duration, const uint8_t* flags, const uint8_t* results,
                    const uint64_t* result_off, uint32_t n, uint32_t* tape, const uint8_t* plan, const uint64_t* body_off, uint8_t* bodies,
                    cudaStream_t s, LaunchLog* lg);
// secret_off: n + 1 absolute uint32 offsets; mac: n x 32 scratch -> n x 71 header characters
cudaError_t wh_sign(const uint8_t* secrets, const uint32_t* secret_off, const uint8_t* flags, const uint8_t* status, const uint8_t* bodies,
                    const uint64_t* body_off, uint32_t n, uint8_t* mac, uint8_t* headers, cudaStream_t s, LaunchLog* lg);
uint64_t wh_fixed_bytes();             // the constant text a body can hold at most

// ---- k_vcworkflow.cu: workflow credentials issued on the device (afc_vcworkflow.cuh).  col_off: 7 absolute offsets per workflow + 1;
// rec_off: n + 1 absolute record indices; rec_col_off (2 per record + 1) and created_at (2 per record) are indexed by absolute record;
// the batch's m = rec_off[n] - rec_off[0] records have per-record scratch cls (m bytes) and id lengths / offsets (m + 1 entries);
// arr: 2 per workflow (where its componentVcIds array starts, its length)
// out: col_off[0], col_off[7 n], rec_off[0], rec_off[n], rec_col_off[2 rec_off[0]], rec_col_off[2 rec_off[n]] (one thread)
cudaError_t vcw_ends(const uint64_t* col_off, const uint64_t* rec_off, const uint64_t* rec_col_off, uint32_t n, uint64_t* out, cudaStream_t s,
                     LaunchLog* lg);
// each record's class and escaped-id length (write them to id_off + 1 for offsets_from_lengths)
cudaError_t vcw_records(const uint8_t* rec_cols, const uint64_t* rec_col_off, const int64_t* created_at, const uint64_t* rec_off, uint32_t m,
                        uint8_t* cls, uint64_t* id_len, cudaStream_t s, LaunchLog* lg);
// each workflow's summary and state, and its signing-message and stored-document length (0 for VCW_HOST; write them to off + 1)
cudaError_t vcw_sizes(const uint8_t* cols, const uint64_t* col_off, const uint64_t* rec_off, const int64_t* created_at, const uint8_t* cls,
                      const uint64_t* id_len, uint32_t n, uint64_t* msg_len, uint64_t* doc_len, uint64_t* arr, uint32_t* summary, uint8_t* state,
                      cudaStream_t s, LaunchLog* lg);
// both byte strings of each workflow's credential around its componentVcIds array; the proofValue is a placeholder until vcw_proof
cudaError_t vcw_fill(const uint8_t* cols, const uint64_t* col_off, const uint64_t* rec_off, const int64_t* created_at, const uint32_t* summary,
                     const uint8_t* state, const uint64_t* arr, uint32_t n, const uint64_t* msg_off, uint8_t* msgs, const uint64_t* doc_off,
                     uint8_t* docs, cudaStream_t s, LaunchLog* lg);
// every record's id into both byte strings (id_off: the scanned id lengths)
cudaError_t vcw_ids(const uint8_t* rec_cols, const uint64_t* rec_col_off, const uint64_t* rec_off, uint32_t n, uint32_t m, const uint8_t* state,
                    const uint64_t* arr, const uint64_t* id_off, const uint64_t* msg_off, uint8_t* msgs, const uint64_t* doc_off, uint8_t* docs,
                    cudaStream_t s, LaunchLog* lg);
// sigs: n x 64, 16-byte aligned -> 86 characters into each built document and into proof_values (zeros for VCW_HOST)
cudaError_t vcw_proof(const uint8_t* sigs, const uint8_t* state, uint32_t n, const uint64_t* doc_off, uint8_t* docs, uint8_t* proof_values,
                      cudaStream_t s, LaunchLog* lg);
uint64_t vcw_literal_bytes();          // constant text of both document forms together

// ---- k_didreg.cu: agent DIDs registered on the device (afc_didreg.cuh).  node_off: n + 1 absolute offsets; id_idx: 2n + 1 absolute id
// indices (request i's reasoners [id_idx[2i], id_idx[2i+1]), skills [id_idx[2i+1], id_idx[2i+2])); id_off: absolute, indexed by absolute id.
// The m = id_idx[2n] - id_idx[0] ids have per-id scratch; the component outputs hold n + m entries (the components, then zeros).
struct DidrArgs {
    const void* comb; const void* ct16;                  // ed_expand_batch's tables (ct16 nullptr: variable-time expansion)
    const uint8_t* master;                               // 32 bytes, 16-byte aligned
    uint32_t h;                                          // didr_server_hash of the server id
    const uint8_t* server; uint64_t server_len;          // the server id's bytes, on the device
    const uint8_t* nodes; const uint64_t* node_off; const uint32_t* agent_index; const uint64_t* id_idx; const uint8_t* ids; const uint64_t* id_off;
    uint32_t n, m;
    // outputs (expanded96, pks, paths 16-byte aligned)
    uint64_t* comp_off; uint8_t* expanded96; uint8_t* pks; uint8_t* dids; uint8_t* paths; uint8_t* comp_flags; uint8_t* body; uint64_t* body_off;
    // scratch: list, flags, esc, rank, before per id; nz m + 1; map_bytes, map_cnt per list; seeds 32 per slot (16-byte aligned);
    // scan json_scan_scratch_bytes(max(n, m))
    uint32_t* list; uint8_t* flags; uint64_t* esc; uint64_t* nz; uint32_t* rank; uint64_t* before; uint64_t* map_bytes; uint32_t* map_cnt;
    uint8_t* seeds; uint64_t* scan;
};
// out: node_off[0], node_off[n], id_idx[0], id_idx[2n], id_off at both (one thread)
cudaError_t didr_ends(const uint64_t* node_off, const uint64_t* id_idx, const uint64_t* id_off, uint32_t n, uint64_t* out, cudaStream_t s,
                      LaunchLog* lg);
// every pass; the seeds scratch holds the derived seeds when it has run (the caller wipes it)
cudaError_t didr_register(const DidrArgs& A, cudaStream_t s, LaunchLog* lg);
uint64_t didr_req_fixed();             // the body bound's constant per request and per id (afc_didreg.cuh)
uint64_t didr_per_id_fixed();

// ---- k_didrereg.cu: known agents re-registered on the device (afc_didrereg.cuh).  agent_col_off: 3n + 1 absolute offsets; id_idx and
// reg_idx: 2n + 1 absolute indices (request i's reasoners [x[2i], x[2i+1]), skills [x[2i+1], x[2i+2])); id_off absolute, indexed by
// absolute id; reg_col_off absolute, component g's five columns at 5g .. 5g + 5.  The m = id_idx[2n] - id_idx[0] ids and the
// G = reg_idx[2n] - reg_idx[0] components have per-item scratch; the key slots are 2n.
struct DidrrArgs {
    const void* comb; const void* ct16;                  // ed_expand_batch's tables (ct16 nullptr: variable-time expansion)
    const uint8_t* master;                               // 32 bytes, 16-byte aligned
    uint32_t h;                                          // didr_server_hash of the server id
    const uint8_t* server; uint64_t server_len;          // the server id's bytes, on the device
    const uint8_t* agent_cols; const uint64_t* agent_col_off; const uint32_t* agent_index;
    const uint64_t* id_idx; const uint8_t* ids; const uint64_t* id_off;
    const uint64_t* reg_idx; const uint8_t* reg_cols; const uint64_t* reg_col_off;
    uint32_t n, m, G;
    // outputs (expanded96, pks, paths 16-byte aligned): per request state, counts (4); per key slot expanded96, pks, dids, paths; per
    // component reg_flags, per id id_flags; the bodies
    uint8_t* state; uint32_t* counts; uint8_t* expanded96; uint8_t* pks; uint8_t* dids; uint8_t* paths; uint8_t* reg_flags; uint8_t* id_flags;
    uint8_t* body; uint64_t* body_off;
    // scratch: rflags, ebytes per component; iflags, esc per id; rank, before per component and id (G + m); bad, agent_bytes per request;
    // map_bytes, map_cnt 4n (the surviving maps, then the new ones); seeds 32 per key slot (16-byte aligned); scan json_scan_scratch_bytes(n)
    uint8_t* rflags; uint64_t* ebytes; uint8_t* iflags; uint64_t* esc; uint32_t* rank; uint64_t* before; uint32_t* bad; uint64_t* agent_bytes;
    uint64_t* map_bytes; uint32_t* map_cnt; uint8_t* seeds; uint64_t* scan;
};
// out: agent_col_off at 0 and 3n, id_idx at 0 and 2n, id_off at both, reg_idx at 0 and 2n, reg_col_off at five times both (one thread)
cudaError_t didrr_ends(const uint64_t* agent_col_off, const uint64_t* id_idx, const uint64_t* id_off, const uint64_t* reg_idx, const uint64_t* reg_col_off,
                       uint32_t n, uint64_t* out, cudaStream_t s, LaunchLog* lg);
// every pass; the seeds scratch holds the derived seeds when it has run (the caller wipes it)
cudaError_t didrr_reregister(const DidrrArgs& A, cudaStream_t s, LaunchLog* lg);
uint64_t didrr_req_fixed();            // the body bound's constant per request and per registered component (afc_didrereg.cuh)
uint64_t didrr_per_reg_fixed();

// ---- k_ed25519.cu
// comb: 32 x 128 ge_precomp (row 0 = the 128 small multiples of B)
size_t ed_tables_bytes();
cudaError_t ed_build_tables(void* comb, cudaStream_t s, LaunchLog* lg);
// Device buffers of the transparent issuer-key cache used by ed_verify_batch (see k_ed25519.cu); owned by afcrypto.cu.
// state words (uint32 each)
enum KcState {
    KS_HIGH = 0,       // ids ever handed out (high-water mark, <= max_keys)
    KS_NHOT = 1,       // credentials of the current call that go through tables
    KS_NCOLD = 2,      // credentials of the current call left to the generic kernel
    KS_DISTINCT = 3,   // distinct public keys in the current call
    KS_NBUILD = 4,     // tables being built in the current call
    KS_EPOCH = 5,      // call counter (LRU stamps)
    KS_NCAND = 6,      // distinct keys of the call that are not cached and are used often enough to deserve a table
    KS_NFREE = 7,      // entries of free_list
    KS_REBUILD = 8,    // the persistent hash table must be rebuilt (something was evicted)
    KS_EVICTED = 9,    // tables evicted in the current call
    KS_TOTAL_BUILT = 10, KS_TOTAL_EVICTED = 11, KS_CALLS = 12,
    KS_QTILE = 13,     // next position of the order the four-lane kernel hands to a warp
    KS_WORDS = 16
};
struct KeyCache {
    // persistent
    uint32_t* slots;        // open-addressing table: slot -> cache id, 0xffffffff = empty   (slot_mask + 1 entries)
    uint32_t slot_mask;
    uint32_t max_keys;
    uint8_t* cpks;          // max_keys x 32
    uint8_t* valid;         // max_keys: key decodes
    void* tabs;             // max_keys x 32 x 128 ge_precomp
    uint32_t* stamp;        // max_keys: epoch of the last call that used the key, 0 = free id
    uint32_t* free_list;    // max_keys: evicted ids waiting for reuse
    uint32_t* bucket;       // max_keys + 1: credentials per id in the current call, then the scatter cursors
    uint32_t* state;        // KS_WORDS
    uint32_t* build_list;   // max_keys: ids whose tables are built in the current call
    void* bases;            // max_keys x 32 x 3 ge_p3: chain output of the tables being built (indexed by build position)
    // per call (capacity >= n)
    uint32_t* bslots;       // batch de-duplication table (bmask + 1 entries, >= 2n)
    uint32_t bmask;
    uint32_t* rep;          // credential -> representative credential (first with the same public key)
    uint32_t* kid;          // representative -> cache id | KC_COLD
    uint32_t* cnt;          // representative -> number of credentials with that key
    uint32_t* dlist;        // distinct representatives
    uint32_t* cand;         // representatives that want a table (at most n / KC_AMORTISE)
    uint32_t* perm;         // hot credentials bucketed by cache id (KS_NHOT entries)
    uint32_t* cold;         // cold credentials (KS_NCOLD entries)
    void* pts;              // 96 bytes per hot position: the projective result of the four-lane kernel, until k_ed_quad_finish
    // the cache work of a call runs on `side` (a high-priority stream) and `side2` between ev_fork and ev_join, while the
    // caller's stream computes H(R||A||M), which does not depend on the cache
    cudaStream_t side, side2;
    cudaEvent_t ev_fork, ev_join, ev_plan, ev_rows, ev_chain[4];
};
cudaError_t ed_keycache_clear(const KeyCache& kc, cudaStream_t s, LaunchLog* lg);     // empties the persistent table (slots, counters)
// scratch_k: n * 32 bytes; kc: nullable (nullptr = always the generic Straus kernel)
cudaError_t ed_verify_batch(const void* comb, const uint8_t* pks, const uint8_t* sigs, const uint8_t* msgs, const uint64_t* off,
                            uint32_t n, uint8_t* ok, uint32_t* scratch_k, const KeyCache* kc, cudaStream_t s, LaunchLog* lg);
size_t ed_key_table_bytes(uint32_t n_keys);
size_t ed_key_bases_bytes(uint32_t n_keys);     // scratch for ed_build_key_tables
cudaError_t ed_build_key_tables(const uint8_t* pks, uint32_t n_keys, void* tabs, uint8_t* valid, void* bases_scratch, cudaStream_t s, LaunchLog* lg);
size_t ed_keyed_scratch_bytes(uint32_t n_keys, uint32_t n);
size_t ed_verify_pts_bytes(uint64_t n);         // KeyCache::pts for a call of n credentials (0 unless AFC_VERIFY_QUAD is set)
// scratch_perm: ed_keyed_scratch_bytes() bytes, 32-byte aligned: projective results, then the issuer-bucketed order (nullptr = credential order, one-thread kernel)
cudaError_t ed_verify_keyed_batch(const void* comb, const void* tabs, const uint8_t* valid, const uint8_t* key_pks, uint32_t n_keys,
                                  const uint32_t* key_index, const uint8_t* sigs, const uint8_t* msgs, const uint64_t* off, uint32_t n,
                                  uint8_t* ok, uint32_t* scratch_k, uint32_t* scratch_perm, cudaStream_t s, LaunchLog* lg);
// ct16: the 48 KB constant-time table (ed_build_ct_table) or nullptr for the fast, variable-time fixed-base multiplication
size_t ed_ct_table_bytes();
cudaError_t ed_build_ct_table(const void* comb, void* ct16, cudaStream_t s, LaunchLog* lg);
cudaError_t ed_sign_batch(const void* comb, const void* ct16, const uint8_t* seeds, const uint8_t* msgs, const uint64_t* off, uint32_t n,
                          uint8_t* sigs, cudaStream_t s, LaunchLog* lg);
// n_keys bounds key_index on the device (an index >= n_keys signs with key 0 instead of reading out of bounds; the host entry
// point has already rejected such a batch, the device-pointer one cannot look)
cudaError_t ed_sign_expanded_batch(const void* comb, const void* ct16, const uint8_t* expanded96, uint32_t n_keys, const uint32_t* key_index,
                                   const uint8_t* msgs, const uint64_t* off, uint32_t n, uint8_t* sigs, cudaStream_t s, LaunchLog* lg);
cudaError_t ed_expand_batch(const void* comb, const void* ct16, const uint8_t* seeds, uint32_t n, uint8_t* expanded96, uint8_t* pks_only,
                            cudaStream_t s, LaunchLog* lg);
// returns number of mismatches in *d_mismatch (device uint32)
cudaError_t ed_selftest(uint32_t iters, uint32_t* d_mismatch, cudaStream_t s, LaunchLog* lg);
cudaError_t microbench_fe(int which, uint32_t iters, uint32_t blocks, uint32_t threads, uint32_t* sink, cudaStream_t s, LaunchLog* lg);

}  // namespace launch
}  // namespace afc
