/* afcrypto.h — C ABI of libafcrypto.so: the H100 (sm_90a) drop-in for AgentField's cryptographic
 * identity-and-audit hot path.  Plain pointers and sizes only; no CUDA or torch types in signatures
 * (streams are passed as void*).  This is exactly what the reference-side cgo adapter binds
 * (INTEGRATION.md shows the Go stubs); each entry point cites the reference code it replaces, relative
 * to /root/reference/control-plane.
 *
 * Conventions
 *   - Batches are PACKED: one contiguous byte buffer + an offsets array of n+1 uint64 (msg i is
 *     bytes [off[i], off[i+1])).  No pointer-to-pointer (cgo cannot pass [][]byte without copying).
 *   - The caller owns every buffer; nothing is retained past return.
 *   - Return 0 on success, negative AFC_E* on failure.  An INVALID SIGNATURE IS NOT AN ERROR: it is
 *     ok[i] = 0 (mirrors how the reference turns failures into Valid:false, vc_service.go:242-289).
 *   - There is NO CPU implementation behind these calls: without a usable CUDA device afc_init fails
 *     with AFC_ECUDA and every other call fails with AFC_EINVAL (NULL ctx).  The reference-side adapter
 *     keeps Go's stdlib as ITS fallback (INTEGRATION.md), not this library.
 *   - Thread-safe and re-entrant: each call takes a stream + staging slot from the ctx pool.
 *   - "_dev" variants take DEVICE pointers and a cudaStream_t (as void*); they only enqueue work.
 */
#ifndef AFCRYPTO_H
#define AFCRYPTO_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)
#endif

#define AFC_OK 0
#define AFC_EINVAL (-1) /* bad argument / bad length (e.g. Go would panic on len(pk) != 32) */
#define AFC_ECUDA (-2)  /* CUDA runtime failure or no device; see afc_last_cuda_error() */
#define AFC_ENOMEM (-3) /* host or device allocation failed */
#define AFC_ENCCL (-4)  /* NCCL failure / NCCL not available */
#define AFC_ESTATE (-5) /* call not valid in the current state */

typedef struct afc_ctx afc_ctx;

/* ---- lifecycle ----------------------------------------------------------------------------------
 * device: CUDA ordinal this context drives (one context per GPU; the control plane shards its pending
 * credential queue round-robin over contexts — SURVEY.md §8e).  Builds the base-point tables on the
 * device. */
int afc_init(int device, afc_ctx** out);
void afc_destroy(afc_ctx* ctx);
const char* afc_strerror(int rc);
const char* afc_last_cuda_error(afc_ctx* ctx);
const char* afc_version(void);
/* device facts for benchmarks: SM count, SM clock kHz, global memory bytes */
int afc_device_info(afc_ctx* ctx, int* sm_count, int* clock_khz, uint64_t* mem_bytes);
/* number of kernel launches issued through this ctx since init (bench "gpu_launches") */
uint64_t afc_launch_count(afc_ctx* ctx);

/* pinned host staging for the adapter's packing buffers (cudaHostAlloc / cudaFreeHost) */
void* afc_alloc_pinned(size_t bytes);
void afc_free_pinned(void* p);
/* the same, but with the pages on the NUMA node of ctx's GPU whichever thread calls (the calling thread is bound to the CPUs in
 * /sys/bus/pci/devices/<gpu>/local_cpulist for the duration of the allocation): what a single process driving several contexts —
 * the Go control plane — uses for its packing pools; the library's own staging buffers are allocated the same way.
 * afc_numa_info: the GPU's NUMA node (-1 if unknown) and the number of CPUs next to it.  AFC_NUMA_BIND=0 disables the binding. */
void* afc_alloc_pinned_for(afc_ctx* ctx, size_t bytes);
int afc_numa_info(afc_ctx* ctx, int* numa_node, int* local_cpus);

/* ---- H1/H2: SHA-256 -----------------------------------------------------------------------------
 * replaces sha256.Sum256 in VCService.hashData (internal/services/vc_service.go:508-515), the
 * streaming digest in FilePayloadStore.SaveFromReader (internal/services/payload_store.go:69-94)
 * and the seed derivation hash (internal/services/did_service.go:515-521).  out32: n x 32 bytes. */
int afc_sha256_batch(afc_ctx* ctx, const uint8_t* msgs, const uint64_t* offsets, uint32_t n, uint8_t* out32);
int afc_sha256_batch_dev(afc_ctx* ctx, const uint8_t* d_msgs, const uint64_t* d_offsets, uint32_t n,
                         uint8_t* d_out32, void* stream);

/* H2 streaming: FilePayloadStore.SaveFromReader (internal/services/payload_store.go:45-97) hashes a payload while it streams to
 * disk, 32 KiB at a time (:154).  Many concurrent uploads = many streams advancing together: stream i absorbs chunk i into its
 * state.  A state is 108 bytes laid out like Go's crypto/sha256 (*digest).MarshalBinary ("sha\x03" || h big-endian || 64-byte
 * buffer || length big-endian) and always sits on a block boundary, so Go code can UnmarshalBinary it and carry on, and back.
 * Every chunk except a stream's last must be a multiple of 64 bytes (the reference's 32 KiB are); where final_flags[i] != 0 the
 * chunk may have any length (also 0), the digest goes to out32[i] and the state is finished.  final_flags may be NULL (none). */
#define AFC_SHA256_STATE_BYTES 108
int afc_sha256_stream_init(uint8_t* states /* n x 108 */, uint32_t n);
int afc_sha256_update_batch(afc_ctx* ctx, uint8_t* states /* n x 108, in/out */, const uint8_t* chunks, const uint64_t* chunk_off /* n+1 */,
                            uint32_t n, const uint8_t* final_flags /* n or NULL */, uint8_t* out32 /* n x 32, written where final */);
int afc_sha256_update_batch_dev(afc_ctx* ctx, uint8_t* d_states, const uint8_t* d_chunks, const uint64_t* d_chunk_off, uint32_t n,
                                const uint8_t* d_final_flags, uint8_t* d_out32, uint8_t* d_status /* n: 0 = malformed state */, void* stream);

/* ---- W1: HMAC-SHA256 ----------------------------------------------------------------------------
 * replaces generateWebhookSignature (internal/services/webhook_dispatcher.go:470-474): tag =
 * HMAC-SHA256(key = secret bytes, msg = body); the "sha256="+hex header text stays host-side.
 * Keys longer than 64 bytes are pre-hashed (RFC 2104, as Go's hmac.New).  key_off: n+1 uint32. */
int afc_hmac_sha256_batch(afc_ctx* ctx, const uint8_t* keys, const uint32_t* key_off, const uint8_t* msgs,
                          const uint64_t* msg_off, uint32_t n, uint8_t* out32);
int afc_hmac_sha256_batch_dev(afc_ctx* ctx, const uint8_t* d_keys, const uint32_t* d_key_off, const uint8_t* d_msgs,
                              const uint64_t* d_msg_off, uint32_t n, uint8_t* d_out32, void* stream);

/* ---- E2: Ed25519 verify -------------------------------------------------------------------------
 * replaces ed25519.Verify in VCService.verifyVCSignature (internal/services/vc_service.go:469-505),
 * verifyWorkflowVCSignature (:1589-1625) and EnhancedVCVerifier.verifyVCSignature
 * (internal/cli/vc_verification_enhanced.go:418-454).  pks: n x 32, sigs: n x 64, ok: n x 1 (0/1).
 * Bit-exact with Go 1.24: S must be canonical, sig[63]&0xE0 must be 0, non-canonical / small-order A
 * accepted, cofactor-less equation, R compared byte-wise with the canonical encoding.
 * (Go panics on len(pk) != 32: the adapter checks lengths before packing and re-panics.) */
int afc_ed25519_verify_batch(afc_ctx* ctx, const uint8_t* pks, const uint8_t* sigs, const uint8_t* msgs,
                             const uint64_t* msg_off, uint32_t n, uint8_t* ok);
int afc_ed25519_verify_batch_dev(afc_ctx* ctx, const uint8_t* d_pks, const uint8_t* d_sigs, const uint8_t* d_msgs,
                                 const uint64_t* d_msg_off, uint32_t n, uint8_t* d_ok, void* stream);

/* Transparent issuer-key cache behind afc_ed25519_verify_batch[_dev]: the batch's public keys are de-duplicated and counted on
 * the device and looked up in a persistent per-context cache of per-key tables (384 KB per key).  The decision is PER KEY:
 * a cached key goes through its table; a key that is not cached but signs at least 48 credentials of the batch gets a table
 * built inside the call (the least recently used tables that this call does not need are evicted when the cache is full);
 * every other credential is verified by the generic kernel in the same call.  Hot credentials are processed bucketed by
 * issuer.  Decisions are taken on the device, nothing synchronises, results are bit-identical whichever way a credential goes.
 * max_keys = 0 disables (always the generic kernel); default 4096 (1.6 GB), or env AFC_KEYCACHE_MAX_KEYS.
 * afc_keycache_info: cached_keys = tables currently held, last_mode = 1 if the last verify call sent any credential through
 * tables.  afc_keycache_stats: the split of the last call and the running totals, and the fixed-base table the table-driven
 * verify reads: base_window = its radix 2^w (16 = the radix-65536 table shared with signing, also what serves when a wider table
 * cannot be allocated), base_table_bytes / base_build_us = the context's verify-only wider table (0 until its first
 * table-driven verify builds it). */
typedef struct afc_keycache_stats_t {
    uint32_t max_keys, cached_keys;
    uint32_t last_hot, last_cold;          /* credentials of the last call verified through tables / by the generic kernel */
    uint32_t last_distinct, last_built, last_evicted;
    uint32_t total_built, total_evicted, calls;
    uint32_t base_window, base_build_us;
    uint64_t base_table_bytes;
} afc_keycache_stats_t;
int afc_keycache_configure(afc_ctx* ctx, uint32_t max_keys);
int afc_keycache_info(afc_ctx* ctx, uint32_t* max_keys, uint32_t* cached_keys, uint32_t* last_mode);
int afc_keycache_stats(afc_ctx* ctx, afc_keycache_stats_t* out);
/* forget every cached table (stream-ordered: enqueued on `stream`, ordered after earlier verify calls); memory is kept */
int afc_keycache_clear(afc_ctx* ctx, void* stream);

/* ---- N1: keyed verification (the identity cache) ---------------------------------------------------------
 * The reference resolves every issuer DID from its own registry before it verifies (VCService.VerifyVC,
 * internal/services/vc_service.go:259 -> DIDService.ResolveDID, internal/services/did_service.go:368-473) and the
 * bulk audit loops over one workflow's VCs (vc_service.go:1442-1512): the verifier knows the key set in advance.
 * afc_keyset_new decodes each key once and builds its radix-256 table of -A on the device (384 KB per key);
 * afc_ed25519_verify_keyed_batch then needs no doublings and no per-credential key decoding (~4.5x fewer field
 * multiplications).  Results are bit-identical to afc_ed25519_verify_batch with pk = keys[key_index[i]]; an index
 * >= n_keys or a key that does not decode yields ok[i] = 0. */
typedef struct afc_keyset afc_keyset;
int afc_keyset_new(afc_ctx* ctx, const uint8_t* pks /* n_keys x 32 */, uint32_t n_keys, afc_keyset** out);
void afc_keyset_free(afc_keyset* ks);
int afc_keyset_info(afc_keyset* ks, uint32_t* n_keys, uint64_t* table_bytes);
int afc_ed25519_verify_keyed_batch(afc_ctx* ctx, afc_keyset* ks, const uint32_t* key_index, const uint8_t* sigs,
                                   const uint8_t* msgs, const uint64_t* msg_off, uint32_t n, uint8_t* ok);
int afc_ed25519_verify_keyed_batch_dev(afc_ctx* ctx, afc_keyset* ks, const uint32_t* d_key_index, const uint8_t* d_sigs,
                                       const uint8_t* d_msgs, const uint64_t* d_msg_off, uint32_t n, uint8_t* d_ok, void* stream);

/* ---- N3: stored credential documents verified on the device ----------------------------------------------------------------
 * replaces, per document, VCService.VerifyVC (internal/services/vc_service.go:242-289: json.Unmarshal :250, ResolveDID :259,
 * verifyVCSignature :469-505 with its zero-Proof json.Marshal :472-476 and base64url decode :498), verifyWorkflowVCSignature
 * (:1589-1625) and EnhancedVCVerifier.verifyVCSignature (internal/cli/vc_verification_enhanced.go:418-454).
 * The device proves that a stored document is byte for byte what json.Marshal writes for the struct (VCDocument / WorkflowVCDocument,
 * pkg/types/did_types.go:135-220) — then the signed message is the document up to "proof": plus the zero proof, built on the device
 * and verified with the key set's tables.  A document it cannot prove canonical is AFC_VC_HOST: the caller parses, re-marshals and
 * verifies that one itself (the Go adapter through its stdlib path), so a verdict is never wrong, a decline only slower.
 * status[i], in the reference's order of errors (parse, resolve, decode signature, verify):
 *   AFC_VC_HOST          not provably canonical: the caller runs Unmarshal -> Marshal -> Verify
 *   AFC_VC_UNRESOLVED    issuer not in the key set ("failed to resolve issuer DID")
 *   AFC_VC_BAD_ENCODING  proofValue is not base64.RawURLEncoding ("failed to decode signature")
 *   AFC_VC_INVALID       ed25519.Verify false, including a decoded signature length other than 64 ("Invalid signature")
 *   AFC_VC_VALID         verified
 * afc_keyset_new_named: afc_keyset_new plus the keys' DIDs (did i = dids[did_off[i] .. did_off[i+1]), n_keys + 1 offsets), looked
 * up by the issuer bytes of each document; a duplicate DID is AFC_EINVAL.  A key set made by afc_keyset_new gives AFC_ESTATE here.
 * fields (NULL or n x 4): issuer offset and length, issuanceDate offset and length as they stand in document i (relative to its
 * start, JSON string bodies without the quotes); valid where status != AFC_VC_HOST.  The host-buffer call streams chunks (documents
 * never straddle one); the _dev call reads doc_off[0] and doc_off[n] once (one synchronisation of `stream`) to size its scratch. */
#define AFC_DOC_EXECUTION_VC 0
#define AFC_DOC_WORKFLOW_VC 1
#define AFC_VC_INVALID 0
#define AFC_VC_VALID 1
#define AFC_VC_HOST 2
#define AFC_VC_UNRESOLVED 3
#define AFC_VC_BAD_ENCODING 4
int afc_keyset_new_named(afc_ctx* ctx, const uint8_t* pks /* n_keys x 32 */, const uint8_t* dids, const uint64_t* did_off /* n_keys+1 */,
                         uint32_t n_keys, afc_keyset** out);
int afc_vc_verify_stored_batch(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* docs, const uint64_t* doc_off, uint32_t n,
                               uint8_t* status, uint32_t* fields);
int afc_vc_verify_stored_batch_dev(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* d_docs, const uint64_t* d_doc_off, uint32_t n,
                                   uint8_t* d_status, uint32_t* d_fields, void* stream);

/* ---- credential documents in any JSON spelling verified on the device ------------------------------------------------------
 * VerifyVC for documents that arrive from outside: request bodies of POST /api/v1/did/verify (internal/handlers/did_handlers.go:97-111)
 * and files given to `af vc verify` (internal/cli/vc.go:159), as the Python SDK (json.dumps), the web UI (JSON.stringify, also
 * pretty-printed) or any other client spells them.  The device reads each document, writes Go's canonical text of it (what
 * json.Marshal(json.Unmarshal(D)) writes, with the zero proof) and verifies that.  Arguments, statuses, fields (spans into the input
 * document), chunking and errors are those of afc_vc_verify_stored_batch; a bad kind or NULL is AFC_EINVAL, a key set without DIDs
 * AFC_ESTATE.  Accepted: whitespace between tokens; every JSON string escape (backslash-u in either case, surrogate pairs), each
 * character re-escaped with Go's rules; int members -?(0|[1-9][0-9]*) up to 18 digits (-0 is 0); metadata values that are strings,
 * true / false / null, integers of up to 15 digits (-0 kept) and arrays / objects up to 8 deep, keys without backslashes in strictly
 * increasing byte order; "errorMessage":"" and "endTime":null (omitted), "endTime":"" (written).  AFC_VC_HOST (the caller runs
 * Unmarshal -> Marshal -> Verify itself) for: member order other than the struct's, missing, unknown, duplicate, re-cased or escaped
 * member names, null for a string, anything that is not JSON (BOM, NaN, trailing commas, raw control bytes, leading zeros),
 * fractions, exponents and longer integers, unsorted or duplicate metadata keys, depth beyond 8, a backslash in issuer or
 * proofValue, raw invalid UTF-8, lone surrogate escapes, and a canonical message longer than the document. */
int afc_vc_verify_json_batch(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* docs, const uint64_t* doc_off, uint32_t n,
                             uint8_t* status, uint32_t* fields);
int afc_vc_verify_json_batch_dev(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* d_docs, const uint64_t* d_doc_off, uint32_t n,
                                 uint8_t* d_status, uint32_t* d_fields, void* stream);

/* ---- VC verification requests answered in one call: POST /api/v1/did/verify (DIDHandlers.VerifyVC, internal/handlers/did_handlers.go:97-111)
 * and POST /api/ui/v1/vc/verify (internal/handlers/ui/did.go:442-469), through VCService.VerifyVC (internal/services/vc_service.go:242-289),
 * for n raw request bodies.  reqs[req_off[i] .. req_off[i+1]) is body i as the client sent it; the call writes state[i], which fixes the HTTP
 * status, and bodies[body_off[i] .. body_off[i+1]), the bytes c.JSON writes (json.Marshal, HTML escaping on, no trailing newline):
 *   AFC_VREQ_OK           200.  json.Marshal(types.VCVerificationResponse) for:
 *                         no vc_document, or a top-level null  {"valid":false,"error":"failed to parse VC document: unexpected end of JSON input"}
 *                         "vc_document":null                   {"valid":false,"error":"failed to resolve issuer DID: DID not found: "}
 *                         an object, the verdict of afc_vc_verify_json_batch on exactly its bytes (AFC_DOC_EXECUTION_VC):
 *                           VALID         {"valid":true,"issuer_did":I,"issued_at":D,"message":"VC verified successfully"}, each of I / D
 *                                         omitted when empty
 *                           INVALID       {"valid":false,"message":"Invalid signature"}
 *                           UNRESOLVED    {"valid":false,"error":"failed to resolve issuer DID: DID not found: " + I}
 *                           BAD_ENCODING  {"valid":false,"error":"failed to verify signature: failed to decode signature: illegal base64 data at
 *                                         input byte " + k}, k the first byte of proofValue outside the URL alphabet, else its last byte
 *   AFC_VREQ_BAD_REQUEST  400.  {"error":"Invalid request body"}: the body holds no JSON value, its first value is not JSON as Go's scanner
 *                         reads it (the whole value is scanned, bytes after it are not), or that value is an array, string, number or bool.
 *                         The UI route adds "details": err.Error() to its 400 body; its caller builds that body itself.
 *   AFC_VREQ_HOST         a zero-length body: the caller runs the handler itself.  A vc_document that is a string, number, array or bool; an
 *                         object afc_vc_verify_json_batch gives AFC_VC_HOST; a null one when the key set holds the DID ""; a top-level
 *                         member name with an escape or a byte >= 0x80; nesting deeper than 64.
 * The member vc_document is matched as Go matches a struct field: the exact name, else any ASCII-case-insensitive spelling; the last one
 * wins.  I and D are the decoded issuer and issuanceDate written with json.Marshal's escaping.  ks is a named key set (afc_keyset_new_named),
 * else AFC_ESTATE.  bodies_cap must be at least afc_vc_verify_request_bound(req_off, n), additive over requests and computed from req_off[0]
 * and req_off[n] alone (a constant per request plus 6 bytes per request byte); else AFC_EINVAL before any work.  Other AFC_EINVAL: a NULL
 * pointer, a key set of another context, a request of 2^31 bytes or more, offsets that run backwards.  The host-buffer call streams chunks
 * of whole requests through the context's staging ring; the _dev call synchronises `stream` once, to read the ends of req_off and whether
 * any request breaks those two rules.  n = 0 writes body_off[0] = 0 in the host-buffer call and nothing in the _dev call. */
#define AFC_VREQ_OK 0
#define AFC_VREQ_BAD_REQUEST 1
#define AFC_VREQ_HOST 2
uint64_t afc_vc_verify_request_bound(const uint64_t* req_off, uint32_t n);
int afc_vc_verify_request_batch(afc_ctx* ctx, afc_keyset* ks, const uint8_t* reqs, const uint64_t* req_off /* n+1 */, uint32_t n,
                                uint8_t* bodies, uint64_t bodies_cap, uint64_t* body_off /* n+1 */, uint8_t* state /* n */);
int afc_vc_verify_request_batch_dev(afc_ctx* ctx, afc_keyset* ks, const uint8_t* d_reqs, const uint64_t* d_req_off, uint32_t n,
                                    uint8_t* d_bodies, uint64_t bodies_cap, uint64_t* d_body_off, uint8_t* d_state, void* stream);

/* ---- stored credentials audited against their records on the device ---------------------------------------------------------
 * replaces, per credential, the checks of VCService.VerifyExecutionVCComprehensive (internal/services/vc_service.go:926-1005):
 * json.Unmarshal, performIntegrityChecks (:1008-1181), performSecurityAnalysis (:1184-1233) and performComplianceChecks
 * (:1236-1268), and of the per-component loop of VerifyWorkflowVCComprehensive (:1442-1512).  Everything afc_vc_verify_stored_batch
 * does (status has the same meaning), plus issues[i], a mask of AFC_AUDIT_* bits for the things the credential has to report:
 *   bits 0-9     the record's column k differs from the document's member (Unmarshal(member) != column; the status column is
 *                compared after NormalizeExecutionStatus on both sides)
 *   INVALID_TIMESTAMP   issuanceDate is not RFC 3339           MISSING_*       validateVCStructure: @context / type empty or null,
 *   NOT_W3C             @context lacks the W3C context                          id / issuer / issuanceDate empty
 *   NOT_AGENTFIELD      type lacks VerifiableCredential or AgentFieldExecutionCredential (workflow documents:
 *                       AgentFieldWorkflowCredential, checkWorkflowVCCompliance :1628-1644; the only bit defined for them)
 *   STATUS_UNDECIDED    the status comparison is left to the caller (non-printable or non-ASCII bytes, or an escape in the document)
 *   TIMESTAMP_UNDECIDED the timestamp rule is left to the caller (a byte >= 0x80 in issuanceDate)
 * issues[i] is 0 and meaningless where status[i] is AFC_VC_HOST.  cols / col_off: AFC_AUDIT_COLUMNS byte strings per record, in the
 * order below, as packed Go strings (column k of record i = cols[col_off[10 i + k] .. col_off[10 i + k + 1]), n * 10 + 1 offsets);
 * required for execution documents, NULL for workflow documents (else AFC_EINVAL).  The host-buffer call streams chunks through
 * the same ring as afc_vc_verify_stored_batch and checks that the column offsets never run backwards; the _dev call synchronises
 * `stream` once to size its scratch. */
#define AFC_AUDIT_COLUMNS 10   /* issuer_did, execution_id, workflow_id, session_id, caller_did, target_did,
                                  status, input_hash, output_hash, signature: the ExecutionVC record, pkg/types */
#define AFC_AUDIT_ISSUER_MISMATCH (1u << 0)
#define AFC_AUDIT_EXECUTION_ID_MISMATCH (1u << 1)
#define AFC_AUDIT_WORKFLOW_ID_MISMATCH (1u << 2)
#define AFC_AUDIT_SESSION_ID_MISMATCH (1u << 3)
#define AFC_AUDIT_CALLER_DID_MISMATCH (1u << 4)
#define AFC_AUDIT_TARGET_DID_MISMATCH (1u << 5)
#define AFC_AUDIT_STATUS_MISMATCH (1u << 6)
#define AFC_AUDIT_INPUT_HASH_MISMATCH (1u << 7)
#define AFC_AUDIT_OUTPUT_HASH_MISMATCH (1u << 8)
#define AFC_AUDIT_SIGNATURE_MISMATCH (1u << 9)
#define AFC_AUDIT_INVALID_TIMESTAMP (1u << 10)
#define AFC_AUDIT_MISSING_CONTEXT (1u << 11)
#define AFC_AUDIT_MISSING_TYPE (1u << 12)
#define AFC_AUDIT_MISSING_ID (1u << 13)
#define AFC_AUDIT_MISSING_ISSUER (1u << 14)
#define AFC_AUDIT_MISSING_ISSUANCE_DATE (1u << 15)
#define AFC_AUDIT_NOT_W3C (1u << 16)
#define AFC_AUDIT_NOT_AGENTFIELD (1u << 17)
#define AFC_AUDIT_STATUS_UNDECIDED (1u << 18)
#define AFC_AUDIT_TIMESTAMP_UNDECIDED (1u << 19)
int afc_vc_audit_stored_batch(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* docs, const uint64_t* doc_off, const uint8_t* cols,
                              const uint64_t* col_off /* n*AFC_AUDIT_COLUMNS+1, NULL for workflow docs */, uint32_t n, uint8_t* status,
                              uint32_t* issues);
int afc_vc_audit_stored_batch_dev(afc_ctx* ctx, afc_keyset* ks, int doc_kind, const uint8_t* d_docs, const uint64_t* d_doc_off, const uint8_t* d_cols,
                                  const uint64_t* d_col_off, uint32_t n, uint8_t* d_status, uint32_t* d_issues, void* stream);

/* ---- E1/K1: Ed25519 sign, public keys -----------------------------------------------------------
 * replaces ed25519.NewKeyFromSeed + ed25519.Sign in VCService.signVC / signWorkflowVC
 * (internal/services/vc_service.go:434-466, :686-718) and NewKeyFromSeed in
 * DIDService.derivePrivateKey (internal/services/did_service.go:515-525).
 * seeds: n x 32; sigs: n x 64 (R || S); pks: n x 32. */
int afc_ed25519_sign_batch(afc_ctx* ctx, const uint8_t* seeds, const uint8_t* msgs, const uint64_t* msg_off,
                           uint32_t n, uint8_t* sigs);
int afc_ed25519_sign_batch_dev(afc_ctx* ctx, const uint8_t* d_seeds, const uint8_t* d_msgs, const uint64_t* d_msg_off,
                               uint32_t n, uint8_t* d_sigs, void* stream);
int afc_ed25519_pubkey_batch(afc_ctx* ctx, const uint8_t* seeds, uint32_t n, uint8_t* pks);
int afc_ed25519_pubkey_batch_dev(afc_ctx* ctx, const uint8_t* d_seeds, uint32_t n, uint8_t* d_pks, void* stream);
/* expanded keys (the N1 identity cache): 96 bytes per key = clamped scalar s (32) || prefix (32) || pk (32).
 * Removes the two redundant fixed-base multiplications the reference does per issued VC
 * (did_service.go:585-599 via ResolveDID, vc_service.go:460). */
int afc_ed25519_expand_batch(afc_ctx* ctx, const uint8_t* seeds, uint32_t n, uint8_t* expanded96);
int afc_ed25519_sign_expanded_batch(afc_ctx* ctx, const uint8_t* expanded96, const uint32_t* key_index,
                                    uint32_t n_keys, const uint8_t* msgs, const uint64_t* msg_off, uint32_t n,
                                    uint8_t* sigs);
int afc_ed25519_expand_batch_dev(afc_ctx* ctx, const uint8_t* d_seeds, uint32_t n, uint8_t* d_expanded96, void* stream);
int afc_ed25519_sign_expanded_batch_dev(afc_ctx* ctx, const uint8_t* d_expanded96, const uint32_t* d_key_index,
                                        const uint8_t* d_msgs, const uint64_t* d_msg_off, uint32_t n,
                                        uint8_t* d_sigs, void* stream);
/* the same with the number of keys stated: an index >= n_keys can then not read key material out of bounds (it signs with key 0;
 * the host-buffer call rejects such a batch with AFC_EINVAL, a device-side index array cannot be inspected without a sync) */
int afc_ed25519_sign_expanded_keys_batch_dev(afc_ctx* ctx, const uint8_t* d_expanded96, uint32_t n_keys, const uint32_t* d_key_index,
                                             const uint8_t* d_msgs, const uint64_t* d_msg_off, uint32_t n, uint8_t* d_sigs, void* stream);

/* Secret scalars (the signing nonce r, and the private scalar when keys are expanded) are multiplied in CONSTANT TIME by default,
 * as Go's crypto/ed25519 does: signed radix 16, a 48 KB table staged in shared memory, every entry of a row read for every digit
 * and one kept by mask — no branch and no address depends on key material.  afc_sign_configure(ctx, 0) (or AFC_SIGN_CT=0) selects
 * the fast variable-time path (radix-65536 table gathers: 16 additions instead of 64) for deployments where nothing untrusted
 * shares the GPU.  Results are identical either way.  Seeds and expanded keys staged by the host-buffer calls are wiped from the
 * device slot and the pinned bounce buffer when the call completes.  afc_sign_mode: 1 = constant time. */
int afc_sign_configure(afc_ctx* ctx, int constant_time);
int afc_sign_mode(afc_ctx* ctx);

/* ---- M1: RFC 6962 Merkle audit log (NEW — the reference's chain check is a stub,
 * internal/cli/vc_verification_enhanced.go:531-534; nearest code generateWorkflowVCDocument,
 * internal/services/vc_service.go:525-632) -----------------------------------------------------------
 * leaf hash = SHA-256(0x00 || leaf), node = SHA-256(0x01 || l || r), split at the largest power of two
 * < n.  The log state (leaf count + <= 64 frontier hashes) lives in a afc_merkle handle on the device.
 * afc_merkle_append adds n leaves and returns the new root and size. */
typedef struct afc_merkle afc_merkle;
int afc_merkle_new(afc_ctx* ctx, afc_merkle** out);
void afc_merkle_free(afc_merkle* m);
int afc_merkle_append(afc_merkle* m, const uint8_t* leaves, const uint64_t* leaf_off, uint32_t n,
                      uint8_t root32[32], uint64_t* tree_size);
int afc_merkle_append_dev(afc_merkle* m, const uint8_t* d_leaves, const uint64_t* d_leaf_off, uint32_t n, void* stream);
/* append n already-hashed nodes (32 bytes each) as leaves-of-this-tree: used to fold per-GPU subtree
 * roots after the all-gather, and to resume a log from stored leaf hashes */
int afc_merkle_append_hashes(afc_merkle* m, const uint8_t* hashes32, uint32_t n, uint8_t root32[32], uint64_t* tree_size);
int afc_merkle_append_hashes_dev(afc_merkle* m, const uint8_t* d_hashes32, uint32_t n, void* stream);
int afc_merkle_root(afc_merkle* m, uint8_t root32[32], uint64_t* tree_size);
int afc_merkle_root_dev(afc_merkle* m, uint8_t* d_root32, void* stream);
/* checkpoint / resume: frontier = up to 64 (height, hash) entries; buffer of 8 + 64*32 bytes */
#define AFC_MERKLE_STATE_BYTES (8 + 64 * 32)
int afc_merkle_save(afc_merkle* m, uint8_t* state);
int afc_merkle_load(afc_merkle* m, const uint8_t* state);
/* one-shot: leaf hashes of a batch (SHA-256(0x00 || leaf)), n x 32 */
int afc_merkle_leaf_hashes_dev(afc_ctx* ctx, const uint8_t* d_leaves, const uint64_t* d_leaf_off, uint32_t n,
                               uint8_t* d_out32, void* stream);

/* ---- E1: issuing execution credentials in one call: GenerateExecutionVC (internal/services/vc_service.go:138-239) for n requests.
 * For request i the call writes exactly what the reference computes and stores:
 *   docs[doc_off[i] .. doc_off[i+1])   the stored vc_document: json.Marshal(createVCDocument(...)) with the signed proof
 *   proof_values[86 i .. 86 i + 86)     the signature (proofValue, base64url without padding)
 *   hashes[86 i .. 86 i + 43), [86 i + 43 .. 86 i + 86)   input_hash and output_hash (hashData: SHA-256 of json.Marshal([]byte),
 *                                       base64url without padding), with AFC_ISSUE_HASH_DATA only (without it both are "")
 * and, with a log, appends the n stored documents (leaf = document bytes) in order, through afc_merkle_append_dev on the call's stream.
 * Inputs:
 *   expanded96 / n_keys / key_index   the issuers' expanded keys (afc_ed25519_expand_batch) and each request's key; signing is constant
 *                                     time unless afc_sign_configure says otherwise
 *   cols / col_off                    AFC_ISSUE_COLUMNS byte strings per request, in the order below (column k of request i =
 *                                     cols[col_off[14 i + k] .. col_off[14 i + k + 1]), n * 14 + 1 absolute offsets).  The VC id,
 *                                     issuanceDate, the proof's created and timestamp are the caller's (the reference reads a clock or
 *                                     makes up an id); error_message is the untruncated message ("" = none)
 *   duration_ms                       n Go ints
 *   payloads / payload_off / payload_nil   2n payloads, input i then output i (payload_off: 2n + 1 absolute offsets; payload_nil[j] != 0
 *                                     for a nil []byte, which hashes as null); read with AFC_ISSUE_HASH_DATA only
 * docs_cap must be at least afc_vc_issue_bound(col_off, n), a bound computed from col_off[0] and col_off[14 n] alone and additive over
 * requests (else AFC_EINVAL, before any work), so a call never fails half-way for lack of room.  Other AFC_EINVAL: a NULL pointer, hashes NULL with
 * AFC_ISSUE_HASH_DATA, unknown flags, n_keys == 0, a log of another context; in the host-buffer call also key_index[i] >= n_keys and
 * offsets that run backwards.  The _dev call cannot inspect its index array without a sync: an index >= n_keys signs with key 0.
 * The host-buffer call streams chunks through the context's staging ring and writes every document at its final offset; the expanded
 * keys it stages are wiped from the device when it returns.  The _dev call synchronises `stream` once, to read the two ends of
 * col_off; expanded96 must be 16-byte aligned.  n = 0 writes doc_off[0] = 0 in the host-buffer call and nothing in the _dev call. */
#define AFC_ISSUE_COLUMNS 14  /* vc_id, caller_did, issuance_date, execution_id, workflow_id, session_id, caller_type,
                                 agent_node_did, target_did, function_name, timestamp, status, error_message, proof_created */
#define AFC_ISSUE_HASH_DATA 1 /* flags: VCRequirements.HashSensitiveData */
uint64_t afc_vc_issue_bound(const uint64_t* col_off, uint32_t n);
int afc_vc_issue_execution_batch(afc_ctx* ctx, const uint8_t* expanded96, uint32_t n_keys, const uint32_t* key_index, const uint8_t* cols,
                                 const uint64_t* col_off /* n*14+1 */, const int64_t* duration_ms, const uint8_t* payloads,
                                 const uint64_t* payload_off /* 2n+1 */, const uint8_t* payload_nil /* 2n */, uint32_t flags, uint32_t n,
                                 afc_merkle* log /* NULL: no append */, uint8_t* docs, uint64_t docs_cap, uint64_t* doc_off /* n+1 */,
                                 uint8_t* hashes /* n x 2 x 43 */, uint8_t* proof_values /* n x 86 */);
int afc_vc_issue_execution_batch_dev(afc_ctx* ctx, const uint8_t* d_expanded96, uint32_t n_keys, const uint32_t* d_key_index, const uint8_t* d_cols,
                                     const uint64_t* d_col_off, const int64_t* d_duration_ms, const uint8_t* d_payloads,
                                     const uint64_t* d_payload_off, const uint8_t* d_payload_nil, uint32_t flags, uint32_t n, afc_merkle* log,
                                     uint8_t* d_docs, uint64_t docs_cap, uint64_t* d_doc_off, uint8_t* d_hashes, uint8_t* d_proof_values,
                                     void* stream);

/* ---- E3: issuing workflow credentials in one call: generateWorkflowVCDocument (internal/services/vc_service.go:525-632), which
 * GetWorkflowVCChain (:292-338) runs on every chain view and VerifyWorkflowVCComprehensive (:1397) on every workflow audit, for n workflows.
 * Workflow i owns records rec_off[i] .. rec_off[i+1] (its ExecutionVC records in GetExecutionVCsByWorkflow order).  The call writes:
 *   docs[doc_off[i] .. doc_off[i+1])   the stored vc_document: json.Marshal(WorkflowVCDocument) with the signed proof; the signature
 *                                       covers the same document with the zero-valued proof (signWorkflowVC).  componentVcIds is always an
 *                                       array ([] without records); totalSteps, completedSteps and metadata.total_executions are the record
 *                                       count; endTime is omitted when nil; issuer, orchestrator.did / agentNodeDid and verificationMethod
 *                                       (+ "#key-1") are the issuer_did column; every column is escaped as Go escapes strings
 *   proof_values[86 i .. 86 i + 86)     the signature (proofValue, base64url without padding)
 *   summary[4 i .. 4 i + 4)             [0] the workflow status (determineWorkflowStatus over NormalizeExecutionStatus of each record, numbered
 *                                       0 unknown, 1 pending, 2 queued, 3 running, 4 succeeded, 5 failed, 6 cancelled, 7 timeout; pending
 *                                       without records), the name the document holds; [1] countCompletedSteps (records whose status
 *                                       normalises to succeeded; the document's completedSteps is the record count, as in the reference);
 *                                       [2] the start record: the first with the earliest (seconds, nanoseconds) (time.Before), relative to
 *                                       rec_off[i]; [3] the end record: the first with the latest time (time.After), 0xFFFFFFFF unless the
 *                                       status is terminal.  Both are 0xFFFFFFFF without records.  The caller takes the full-precision StartTime
 *                                       and EndTime from those records; the document holds them as UTC().Format(time.RFC3339).
 *   state[i]                            AFC_WORKFLOW_BUILT, or AFC_WORKFLOW_HOST: a zero-length document, a zeroed proof value and summary;
 *                                       the caller builds that workflow itself.  HOST: a record status with a byte outside printable ASCII
 *                                       and \t \n \v \f \r (Go's TrimSpace / ToLower are Unicode-aware), a created_at outside
 *                                       0001-01-01T00:00:00Z .. 9999-12-31T23:59:59Z, or nanoseconds outside [0, 10^9).
 * Deviation: without records the reference reads time.Now() for startTime, then again for snapshotTime; this call writes the snapshot_time
 * column's text for both.
 * Inputs:
 *   expanded96 / n_keys / key_index   the issuers' expanded keys and each workflow's key (issuer_did's); signing is constant time unless
 *                                     afc_sign_configure says otherwise
 *   cols / col_off                    AFC_WORKFLOW_COLUMNS byte strings per workflow, n * 7 + 1 absolute offsets.  session_id and issuer_did
 *                                     are the first record's (issuer_did: the root DID without records); vc_id, issuance_date, snapshot_time
 *                                     and proof_created are the caller's (the reference makes up an id and reads a clock)
 *   rec_off                           n + 1 absolute record indices, non-decreasing
 *   rec_cols / rec_col_off            AFC_WORKFLOW_RECORD_COLUMNS byte strings per record; record r's column k is
 *                                     rec_cols[rec_col_off[2 r + k] .. rec_col_off[2 r + k + 1])
 *   created_at                        2 int64 per record (created_at[2 r], [2 r + 1]): CreatedAt as Unix seconds and nanoseconds
 * docs_cap must be at least afc_vc_workflow_bound(col_off, rec_off, rec_col_off, n), computed from the ends of the three offset arrays
 * alone and additive over workflows (else AFC_EINVAL, before any work).  Other AFC_EINVAL: a NULL pointer, n_keys == 0; in the host-buffer
 * call also key_index[i] >= n_keys and offsets that run backwards.  The _dev call cannot inspect its index array without a sync: an index
 * >= n_keys signs with key 0.  The host-buffer call streams chunks of whole workflows through the context's staging ring (a workflow
 * bigger than a slot goes alone) and writes every document at its final offset; the expanded keys it stages are wiped from the device
 * when it returns.  The _dev call synchronises `stream` once, to read the ends of the offset arrays; expanded96 must be 16-byte aligned
 * there.  n = 0 writes doc_off[0] = 0 in the host-buffer call and nothing in the _dev call.  Nothing is logged: the reference
 * neither persists nor logs these snapshots. */
#define AFC_WORKFLOW_COLUMNS 7         /* workflow_id, session_id, issuer_did, vc_id, issuance_date, snapshot_time, proof_created */
#define AFC_WORKFLOW_RECORD_COLUMNS 2  /* vc_id, status of each ExecutionVC record, in GetExecutionVCsByWorkflow order */
#define AFC_WORKFLOW_BUILT 0
#define AFC_WORKFLOW_HOST 1
uint64_t afc_vc_workflow_bound(const uint64_t* col_off, const uint64_t* rec_off, const uint64_t* rec_col_off, uint32_t n);
int afc_vc_issue_workflow_batch(afc_ctx* ctx, const uint8_t* expanded96, uint32_t n_keys, const uint32_t* key_index /* n */, const uint8_t* cols,
                                const uint64_t* col_off /* 7n+1 */, const uint64_t* rec_off /* n+1 absolute record indices */,
                                const uint8_t* rec_cols, const uint64_t* rec_col_off /* 2 per record +1 */,
                                const int64_t* created_at /* per record: Unix seconds, nanoseconds */, uint32_t n, uint8_t* docs, uint64_t docs_cap,
                                uint64_t* doc_off /* n+1 */, uint8_t* proof_values /* n x 86 */, uint8_t* state /* n */, uint32_t* summary /* n x 4 */);
int afc_vc_issue_workflow_batch_dev(afc_ctx* ctx, const uint8_t* d_expanded96, uint32_t n_keys, const uint32_t* d_key_index, const uint8_t* d_cols,
                                    const uint64_t* d_col_off, const uint64_t* d_rec_off, const uint8_t* d_rec_cols, const uint64_t* d_rec_col_off,
                                    const int64_t* d_created_at, uint32_t n, uint8_t* d_docs, uint64_t docs_cap, uint64_t* d_doc_off,
                                    uint8_t* d_proof_values, uint8_t* d_state, uint32_t* d_summary, void* stream);

/* ---- E4: workflow VC chains served in one call: GetWorkflowVCChain (internal/services/vc_service.go:292-338) with
 * collectDIDResolutionBundle (:810-870) and the handler's c.JSON (internal/handlers/ui/did.go:383), for n workflows.
 * afc_did_directory_new: the registry's public half — n DIDs (did i = dids[did_off[i] .. did_off[i+1]), n + 1 offsets) and their public
 * keys (pks, n x 32), looked up as a named key set looks up its DIDs, with each DID's rank in byte order (strings.Compare) computed once.
 * No verify tables are built, so a directory of 10^6 DIDs takes tens of MB.  A duplicate DID, a NULL pointer or offsets that run
 * backwards give AFC_EINVAL.
 * afc_vc_workflow_chain_batch writes, for workflow i, bodies[body_off[i] .. body_off[i+1]): json.Marshal(types.WorkflowVCChainResponse),
 * HTML escaping on, byte for byte, and state[i]:
 *   AFC_CHAIN_BUILT   the body
 *   AFC_CHAIN_HOST    a zero-length body; the caller builds it itself.  HOST covers every AFC_WORKFLOW_HOST workflow of the issue call;
 *                     a non-nil vc_document that is empty or not JSON (json.Marshal fails in Go), or nested deeper than 32; a created_at
 *                     or snapshot time whose UTC offset is not a whole number of minutes or is 24 hours or more, or whose local year
 *                     falls outside 1..9999; a resolved_at column longer than 64 bytes; a DID longer than 128 bytes that the bundle would hold.
 * The body: component_vcs holds each record in ExecutionVC field order, agent_node_id / workflow_name omitted when nil, vc_document
 * compacted as Go's appendCompact does (whitespace outside strings dropped; < > & U+2028 U+2029 escaped), null when nil, created_at as
 * Time.MarshalJSON writes it; parent_vc_id and child_vc_ids are never set by storage (vc_storage.go:234-263), so they are never written.
 * workflow_vc is the credential afc_vc_issue_workflow_batch issues on the same inputs (vc_document, signature = its proof value), with
 * start_time / end_time at full precision from the records summary[2] / [3] names, in their own offsets, and snapshot_time from the clock.
 * did_resolution_bundle holds the issuer, caller and target DIDs of every record and the credential's issuer, without "", "did:key:" and
 * DIDs strings.TrimSpace empties, that the directory holds, once each, in byte order; each with its method (strings.Split(did, ":")[1]
 * after a "did:" prefix and more, "key" otherwise), the public JWK ed25519PublicKeyToJWK writes for the directory's key, "bundled" and
 * resolved_at.  The member is omitted when the bundle is empty.
 * Inputs: every argument of afc_vc_issue_workflow_batch, unchanged, and
 *   chain_cols / chain_col_off      AFC_CHAIN_WORKFLOW_COLUMNS byte strings per workflow, 2n + 1 absolute offsets
 *   clock                           3 int64 per workflow: the snapshot time as Unix seconds, nanoseconds and UTC offset in seconds; also
 *                                   StartTime of a workflow without records (the reference reads time.Now() for both)
 *   chain_rec_cols / chain_rec_col_off   AFC_CHAIN_RECORD_COLUMNS byte strings per record, indexed by absolute record as rec_col_off
 *   rec_flags                       per record: AFC_CHAIN_AGENT_NODE_ID_NIL, AFC_CHAIN_WORKFLOW_NAME_NIL, AFC_CHAIN_VC_DOCUMENT_NIL
 *   doc_size                        per record: document_size_bytes
 *   created_off                     per record: the UTC offset of created_at in seconds
 * bodies_cap must be at least afc_vc_workflow_chain_bound(...), computed from the ends of the five offset arrays alone and additive over
 * workflows (else AFC_EINVAL, before any work).  Other AFC_EINVAL: a NULL pointer, n_keys == 0, a directory of another context, more
 * than 2^31 - 1 DID occurrence slots (3 per record, 1 per workflow); in the host-buffer call also key_index[i] >= n_keys and offsets
 * that run backwards.  The host-buffer call streams chunks of whole workflows through the context's staging ring; the expanded keys it
 * stages are wiped from the device when it returns.  The _dev call synchronises `stream` once, to read the ends of the offset arrays; expanded96 must be 16-byte aligned there.
 * n = 0 writes body_off[0] = 0 in the host-buffer call and nothing in the _dev call. */
typedef struct afc_did_directory afc_did_directory;
int afc_did_directory_new(afc_ctx* ctx, const uint8_t* pks /* n x 32 */, const uint8_t* dids, const uint64_t* did_off /* n+1 */, uint32_t n,
                          afc_did_directory** out);
void afc_did_directory_free(afc_did_directory* dir);
#define AFC_CHAIN_WORKFLOW_COLUMNS 2   /* workflow_vc_id, resolved_at */
#define AFC_CHAIN_RECORD_COLUMNS 13    /* execution_id, workflow_id, session_id, agent_node_id, workflow_name, issuer_did, target_did,
                                          caller_did, vc_document, signature, storage_uri, input_hash, output_hash */
#define AFC_CHAIN_AGENT_NODE_ID_NIL 1
#define AFC_CHAIN_WORKFLOW_NAME_NIL 2
#define AFC_CHAIN_VC_DOCUMENT_NIL 4
#define AFC_CHAIN_BUILT 0
#define AFC_CHAIN_HOST 1
uint64_t afc_vc_workflow_chain_bound(const uint64_t* col_off, const uint64_t* rec_off, const uint64_t* rec_col_off, const uint64_t* chain_col_off,
                                     const uint64_t* chain_rec_col_off, uint32_t n);
int afc_vc_workflow_chain_batch(afc_ctx* ctx, const uint8_t* expanded96, uint32_t n_keys, const uint32_t* key_index, const uint8_t* cols,
                                const uint64_t* col_off, const uint64_t* rec_off, const uint8_t* rec_cols, const uint64_t* rec_col_off,
                                const int64_t* created_at, const uint8_t* chain_cols, const uint64_t* chain_col_off /* 2n+1 */,
                                const int64_t* clock /* 3n */, const uint8_t* chain_rec_cols, const uint64_t* chain_rec_col_off /* 13 per record +1 */,
                                const uint8_t* rec_flags, const int64_t* doc_size, const int32_t* created_off, const afc_did_directory* dir, uint32_t n,
                                uint8_t* bodies, uint64_t bodies_cap, uint64_t* body_off /* n+1 */, uint8_t* state /* n */);
int afc_vc_workflow_chain_batch_dev(afc_ctx* ctx, const uint8_t* d_expanded96, uint32_t n_keys, const uint32_t* d_key_index, const uint8_t* d_cols,
                                    const uint64_t* d_col_off, const uint64_t* d_rec_off, const uint8_t* d_rec_cols, const uint64_t* d_rec_col_off,
                                    const int64_t* d_created_at, const uint8_t* d_chain_cols, const uint64_t* d_chain_col_off, const int64_t* d_clock,
                                    const uint8_t* d_chain_rec_cols, const uint64_t* d_chain_rec_col_off, const uint8_t* d_rec_flags,
                                    const int64_t* d_doc_size, const int32_t* d_created_off, const afc_did_directory* dir, uint32_t n,
                                    uint8_t* d_bodies, uint64_t bodies_cap, uint64_t* d_body_off, uint8_t* d_state, void* stream);

/* ---- N1: DIDs resolved and W3C DID documents served in one call: DIDService.ResolveDID (internal/services/did_service.go:368-473) and
 * the c.JSON of GET /api/v1/did/resolve/:did and GET /api/v1/did/document/:did (internal/handlers/did_handlers.go:73-94, 368-429), for n
 * requests against a directory.  The handlers' registry checks (DID system disabled, no server registry) stay with the caller.
 * afc_did_directory_set_identities gives each directory DID, in the order given to afc_did_directory_new, its kind (AFC_DID_KIND_*) and
 * three byte strings: derivation_path, function_name, public_key_jwk (the stored JWK text; for the root, ed25519PublicKeyToJWK's text of
 * its key); cols / col_off: 3n + 1 absolute offsets, DID k's strings at col_off[3k .. 3k + 3].  One pass on the device computes each
 * entry's two body lengths, or HOST, and the directory's longest body.  AFC_EINVAL: a NULL pointer, a kind above AFC_DID_KIND_SKILL,
 * offsets that run backwards, a directory that already has identities.  A directory without identities serves
 * afc_vc_workflow_chain_batch as before.
 * afc_did_resolve_batch writes, for request i = (kinds[i], reqs[req_off[i] .. req_off[i+1])), bodies[body_off[i] .. body_off[i+1]): the
 * bytes c.JSON writes (json.Marshal, HTML escaping on, map keys sorted), and state[i], which fixes the HTTP status:
 *   AFC_DIDRES_FOUND        200.  RESOLVE: {"component_type","derivation_path","did","function_name","public_key_jwk"}, the JWK as a
 *                           JSON string; component_type "agentfield_server", "agent", "reasoner" or "skill" from the kind.  DOCUMENT: the
 *                           W3C DID document of did_handlers.go:398-425, publicKeyJwk the stored JWK re-marshalled through
 *                           map[string]interface{} (keys sorted, numbers as float64, strings re-escaped; a stored null stays null).
 *   AFC_DIDRES_NOT_FOUND    404.  {"error":"DID not found"}, or for DOCUMENT {"details":"DID not found: <the request, escaped>","error":...}.
 *   AFC_DIDRES_BAD_REQUEST  400.  An empty DID: {"error":"DID parameter is required"}.
 *   AFC_DIDRES_HOST         a zero-length body; the caller builds it.  A DOCUMENT whose stored JWK json.Unmarshal rejects or holds a
 *                           value other than an object or null (a 500 in the reference), or one the device does not re-marshal (duplicate
 *                           or escaped keys, invalid UTF-8 or lone surrogates, nesting deeper than 32, numbers outside float64's normal
 *                           range); either kind when the found body would exceed 4096 bytes; a kind other than RESOLVE and DOCUMENT.
 * bodies_cap must be at least afc_did_resolve_bound(dir, req_off, n), additive over requests and computed from the directory and the ends
 * of req_off alone (else AFC_EINVAL, before any work).  Other AFC_EINVAL: a NULL pointer, a directory without identities or of another
 * context, a request of 2^31 bytes or more, offsets that run backwards.  The host-buffer call streams chunks of whole requests through
 * the context's staging ring; the _dev call synchronises `stream` once, to read the ends of req_off and whether any request breaks those
 * two rules.  n = 0 writes body_off[0] = 0 in the host-buffer call and nothing in the _dev call.  No secret is involved: the call derives
 * no key and does not rebuild the private JWK ResolveDID regenerates and both handlers discard. */
#define AFC_DID_KIND_SERVER 0
#define AFC_DID_KIND_AGENT 1
#define AFC_DID_KIND_REASONER 2
#define AFC_DID_KIND_SKILL 3
#define AFC_DID_IDENTITY_COLUMNS 3   /* derivation_path, function_name, public_key_jwk */
#define AFC_DIDRES_RESOLVE 0
#define AFC_DIDRES_DOCUMENT 1
#define AFC_DIDRES_FOUND 0
#define AFC_DIDRES_NOT_FOUND 1
#define AFC_DIDRES_BAD_REQUEST 2
#define AFC_DIDRES_HOST 3
int afc_did_directory_set_identities(afc_did_directory* dir, const uint8_t* kinds /* n */, const uint8_t* cols, const uint64_t* col_off /* 3n+1 */);
uint64_t afc_did_resolve_bound(const afc_did_directory* dir, const uint64_t* req_off, uint32_t n);
int afc_did_resolve_batch(afc_ctx* ctx, const afc_did_directory* dir, const uint8_t* kinds, const uint8_t* reqs, const uint64_t* req_off /* n+1 */,
                          uint32_t n, uint8_t* bodies, uint64_t bodies_cap, uint64_t* body_off /* n+1 */, uint8_t* state /* n */);
int afc_did_resolve_batch_dev(afc_ctx* ctx, const afc_did_directory* dir, const uint8_t* d_kinds, const uint8_t* d_reqs, const uint64_t* d_req_off,
                              uint32_t n, uint8_t* d_bodies, uint64_t bodies_cap, uint64_t* d_body_off, uint8_t* d_state, void* stream);

/* ---- W2: execution webhook deliveries built and signed in one call: determineWebhookEvent + buildPayload + json.Marshal +
 * generateWebhookSignature (internal/services/webhook_dispatcher.go:294-320, 394-474) for n deliveries.  For delivery i:
 *   bodies[body_off[i] .. body_off[i+1])   the request body json.Marshal(types.ExecutionWebhookPayload), the result member being
 *                                        json.Marshal(json.Unmarshal(raw)) (map keys sorted, numbers as float64, strings re-escaped)
 *                                        or, for raw the JSON grammar rejects, the string(raw)
 *   headers[71 i .. 71 i + 71)           the X-AgentField-Signature value "sha256=" + hex(HMAC-SHA256(secret, body)) with
 *                                        AFC_WEBHOOK_HAS_SECRET, 71 zero bytes without
 *   status[i]                            AFC_WEBHOOK_BUILT, or AFC_WEBHOOK_HOST: a zero-length body and a zeroed header; the caller
 *                                        builds that delivery itself.  HOST: a status that is not printable ASCII (the event rule), and a
 *                                        result the device does not re-marshal exactly (duplicate or escaped keys, invalid UTF-8 or lone
 *                                        surrogate escapes, nesting beyond 32 levels, numbers outside the normal float64 range, an
 *                                        Eisel-Lemire give-up)
 * Inputs:
 *   cols / col_off     AFC_WEBHOOK_COLUMNS byte strings per delivery in the order below, n * 8 + 1 absolute offsets.  target_type is the
 *                      caller's resolveTargetType; timestamp is the caller's RFC 3339 text (CompletedAt, or now)
 *   duration_ms        n int64, read with AFC_WEBHOOK_HAS_DURATION (else the member is omitted; 0 is written)
 *   flags              n bytes of AFC_WEBHOOK_HAS_*; error_message is written for the failed event with AFC_WEBHOOK_HAS_ERROR_MESSAGE only
 *   results / result_off   the stored ResultPayload of each delivery, n + 1 absolute offsets (empty = nil)
 *   secrets / secret_off   the webhook secrets, n + 1 absolute uint32 offsets (read with AFC_WEBHOOK_HAS_SECRET only; any length)
 * results and secrets may be NULL in the host-buffer call when their offsets span no bytes (results also in the _dev call).
 * bodies_cap must be at least afc_webhook_bound(col_off, result_off, n), computed from the two ends of both offset arrays alone and
 * additive over deliveries (else AFC_EINVAL before any work).  Other AFC_EINVAL: a NULL pointer, unknown flag bits (host-buffer call),
 * offsets that run backwards (host-buffer call).  The host-buffer call streams chunks through the context's staging ring, writes every
 * body at its final offset and wipes the staged secrets from the device slot and the pinned bounce buffer when it returns.  The _dev
 * call synchronises `stream` once, to read the ends of col_off and result_off.  n = 0 writes body_off[0] = 0 in the host-buffer call
 * and nothing in the _dev call. */
#define AFC_WEBHOOK_COLUMNS 8   /* execution_id, run_id, status, node_id, reasoner_id, target_type, timestamp, error_message */
#define AFC_WEBHOOK_HAS_DURATION 1
#define AFC_WEBHOOK_HAS_ERROR_MESSAGE 2
#define AFC_WEBHOOK_HAS_SECRET 4
#define AFC_WEBHOOK_BUILT 0
#define AFC_WEBHOOK_HOST 1
#define AFC_WEBHOOK_HEADER_CHARS 71
uint64_t afc_webhook_bound(const uint64_t* col_off, const uint64_t* result_off, uint32_t n);
int afc_webhook_sign_batch(afc_ctx* ctx, const uint8_t* cols, const uint64_t* col_off /* n*8+1 */, const int64_t* duration_ms, const uint8_t* flags,
                           const uint8_t* results, const uint64_t* result_off /* n+1 */, const uint8_t* secrets, const uint32_t* secret_off /* n+1 */,
                           uint32_t n, uint8_t* bodies, uint64_t bodies_cap, uint64_t* body_off /* n+1 */, uint8_t* headers /* n x 71 */,
                           uint8_t* status /* n */);
int afc_webhook_sign_batch_dev(afc_ctx* ctx, const uint8_t* d_cols, const uint64_t* d_col_off, const int64_t* d_duration_ms, const uint8_t* d_flags,
                               const uint8_t* d_results, const uint64_t* d_result_off, const uint8_t* d_secrets, const uint32_t* d_secret_off,
                               uint32_t n, uint8_t* d_bodies, uint64_t bodies_cap, uint64_t* d_body_off, uint8_t* d_headers, uint8_t* d_status,
                               void* stream);

/* ---- K1/K2: agent DIDs registered in one call: handleNewRegistration (internal/services/did_service.go:186-365) for n new agents.
 * For request i, its components are comp_off[i] .. comp_off[i+1]: the agent, then its non-empty reasoner ids in request order, then its
 * non-empty skill ids.  Paths: agent m/44'/<h>'/<a>', reasoner m/44'/<h>'/<a>'/0'/<j>', skill m/44'/<h>'/<a>'/1'/<j>', where h =
 * FNV-1a 32(server_id) mod 2^31, a = agent_index[i] and j counts the non-empty ids before this one in its list.  Component c:
 *   expanded96[96 c ..]   ed25519.NewKeyFromSeed(SHA-256(master_seed || path)) as afc_ed25519_expand_batch writes it (s || prefix || pk),
 *                         ready for afc_ed25519_sign_expanded* and both issue calls
 *   pks[32 c ..]          the public key
 *   dids[55 c ..]         did:key:z + base64url(0xED 0x01 || pk)
 *   paths[48 c ..]        the derivation path, NUL-padded (at most 44 bytes)
 *   comp_flags[c]         AFC_DID_KEPT: in the identity package (and the registry); clear for an id repeated later in its list, whose
 *                         later occurrence the map keeps
 * and body[body_off[i] .. body_off[i+1]) is json.Marshal(types.DIDRegistrationResponse), the bytes the registration handler writes: every
 * kept component's identity with its private and public JWK, maps keyed by the raw ids in byte order, the server id and the message.
 * Inputs:
 *   master_seed              the registry's 32-byte master seed (a device pointer in the _dev call, 16-byte aligned)
 *   server_id / _len         the server id (a host pointer in both calls)
 *   node_ids / node_off      each request's agent_node_id, n + 1 absolute offsets
 *   agent_index              n values: len(registry.AgentNodes) when the request is handled (the caller keeps the registry)
 *   id_idx                   2n + 1 absolute id indices: request i's reasoner ids are [id_idx[2i], id_idx[2i+1]), its skill ids
 *                            [id_idx[2i+1], id_idx[2i+2]); id k is ids[id_off[k] .. id_off[k+1])
 * The component outputs hold n + m entries, m = id_idx[2n] - id_idx[0]: the comp_off[n] components, then zeros.  body_cap must be at
 * least afc_did_register_bound(node_off, id_idx, id_off, n, server_id_len), computed from the ends of the three offset arrays and additive
 * over requests (else AFC_EINVAL, before any work).  Other AFC_EINVAL: a NULL pointer, more than 2^32 - 1 components; in the host-buffer call
 * also offsets that run backwards.  The host-buffer call runs chunks of whole requests, one after another, through one of the context's
 * staging slots (a request bigger than a chunk's budget goes alone) and wipes every secret it staged there, the master seed and the
 * bodies included, whatever the outcome.  The _dev call synchronises `stream` once, to read the ends of the offset arrays; expanded96, pks and
 * paths must be 16-byte aligned there.  Derived seeds and expanded keys are wiped from every device scratch area before either call returns:
 * the caller's outputs are the only place they remain.  The expansion is constant time unless afc_sign_configure says otherwise.  n = 0
 * writes comp_off[0] = body_off[0] = 0 in the host-buffer call and nothing in the _dev call. */
#define AFC_DID_CHARS 55
#define AFC_DID_PATH_SLOT 48
#define AFC_DID_KEPT 1
uint64_t afc_did_register_bound(const uint64_t* node_off, const uint64_t* id_idx, const uint64_t* id_off, uint32_t n, uint64_t server_id_len);
int afc_did_register_batch(afc_ctx* ctx, const uint8_t* master_seed /* 32 */, const uint8_t* server_id, uint64_t server_id_len,
                           const uint8_t* node_ids, const uint64_t* node_off /* n+1 */, const uint32_t* agent_index /* n */,
                           const uint64_t* id_idx /* 2n+1 */, const uint8_t* ids, const uint64_t* id_off, uint32_t n, uint64_t* comp_off /* n+1 */,
                           uint8_t* expanded96, uint8_t* pks, uint8_t* dids, uint8_t* paths, uint8_t* comp_flags, uint8_t* body, uint64_t body_cap,
                           uint64_t* body_off /* n+1 */);
int afc_did_register_batch_dev(afc_ctx* ctx, const uint8_t* d_master_seed, const uint8_t* server_id, uint64_t server_id_len, const uint8_t* d_node_ids,
                               const uint64_t* d_node_off, const uint32_t* d_agent_index, const uint64_t* d_id_idx, const uint8_t* d_ids,
                               const uint64_t* d_id_off, uint32_t n, uint64_t* d_comp_off, uint8_t* d_expanded96, uint8_t* d_pks, uint8_t* d_dids,
                               uint8_t* d_paths, uint8_t* d_comp_flags, uint8_t* d_body, uint64_t body_cap, uint64_t* d_body_off, void* stream);

/* ---- K3: known agents re-registered in one call: RegisterAgent's branch for an agent the registry holds (internal/services/
 * did_service.go:154-179): PerformDifferentialAnalysis (:757-847), then buildExistingIdentityPackage (:940-986) when nothing changed,
 * DeregisterComponents (:1239-1324) for the removed components, and PartialRegisterAgent (:1049-1236) for the new ones.  The call holds
 * no registry: the caller passes each agent's record and applies the flags below to its registry.
 * Inputs per request i (strings as in afc_did_register_batch: packed bytes and absolute offsets):
 *   master_seed / server_id      as in afc_did_register_batch
 *   agent_cols / agent_col_off   3 strings per request (3n + 1 offsets): the stored did, public_key_jwk and derivation_path of the agent
 *   agent_index                  n values: the <a> of the new components' paths m/44'/<h>'/<a>'/<0|1>'/<j>'.  The reference takes the
 *                                agent's place in Go's randomised iteration over the registry; a stable choice is the <a> of the agent's
 *                                own stored derivation path
 *   id_idx / ids / id_off        the request's reasoner and skill ids, laid out as in afc_did_register_batch
 *   reg_idx / reg_cols / reg_col_off   the registered components: request i's reasoners are [reg_idx[2i], reg_idx[2i+1]), its skills
 *                                [reg_idx[2i+1], reg_idx[2i+2]); component g has 5 strings at reg_col_off[5g .. 5g+5]: its map key, did,
 *                                stored public_key_jwk, derivation_path and function_name
 * Outputs per request:
 *   state[i]        AFC_DIDRR_UNCHANGED (nothing new or removed), AFC_DIDRR_REMOVED (removals only), AFC_DIDRR_PARTIAL (new components),
 *                   AFC_DIDRR_INVALID (a registered list holds one key twice, which no Go map can: refused, with an empty body, zero
 *                   counts, flags and key slots)
 *   counts[4i ..]   new reasoners, new skills (distinct ids: the maps' sizes), removed reasoners, removed skills
 *   body[body_off[i] .. body_off[i+1])   json.Marshal(types.DIDRegistrationResponse): for UNCHANGED and REMOVED the existing identity package
 *                   of the surviving components (every private_key_jwk "", public_key_jwk as stored, function_name omitted when empty);
 *                   for PARTIAL only the new components, each with its private JWK; the agent's own identity always as stored
 *   key slots 2i + kind (kind 0 reasoners, 1 skills): expanded96[96 ..], pks[32 ..], dids[55 ..], paths[48 ..] of the one key every new
 *                   component of that kind receives (its path index j is the map's size after the removals, as in the reference); zeros
 *                   where the request adds none
 * Outputs per component and id:
 *   reg_flags[g - reg_idx[0]]   AFC_DIDRR_GONE: DeregisterComponents removes it
 *   id_flags[r - id_idx[0]]     AFC_DIDRR_NEW for a new id, with AFC_DID_KEPT on the occurrence the map keeps (the last)
 * The caller's registry update: delete the GONE components, then add each NEW + KEPT id with its slot's DID, path and public key.
 * body_cap must be at least afc_did_reregister_bound(...), computed from the ends of the five offset arrays and additive over requests (else
 * AFC_EINVAL, before any work).  Other AFC_EINVAL: a NULL pointer, more than 2^32 - 1 ids, components or key slots; in the host-buffer call
 * also offsets that run backwards.  Naming one node twice in a batch has no defined result (the reference handles requests one after
 * another): the caller must not.  Chunking, secrets (the master seed, derived seeds, expanded keys and bodies are wiped from staging
 * memory), alignment, the single synchronisation of the _dev call and n = 0 are as in afc_did_register_batch. */
#define AFC_DIDRR_UNCHANGED 0
#define AFC_DIDRR_REMOVED 1
#define AFC_DIDRR_PARTIAL 2
#define AFC_DIDRR_INVALID 3
#define AFC_DIDRR_GONE 1
#define AFC_DIDRR_NEW 2
uint64_t afc_did_reregister_bound(const uint64_t* agent_col_off, const uint64_t* id_idx, const uint64_t* id_off, const uint64_t* reg_idx,
                                  const uint64_t* reg_col_off, uint32_t n, uint64_t server_id_len);
int afc_did_reregister_batch(afc_ctx* ctx, const uint8_t* master_seed /* 32 */, const uint8_t* server_id, uint64_t server_id_len,
                             const uint8_t* agent_cols, const uint64_t* agent_col_off /* 3n+1 */, const uint32_t* agent_index /* n */,
                             const uint64_t* id_idx /* 2n+1 */, const uint8_t* ids, const uint64_t* id_off, const uint64_t* reg_idx /* 2n+1 */,
                             const uint8_t* reg_cols, const uint64_t* reg_col_off, uint32_t n, uint8_t* state /* n */, uint32_t* counts /* 4n */,
                             uint8_t* expanded96 /* 2n x 96 */, uint8_t* pks /* 2n x 32 */, uint8_t* dids /* 2n x 55 */, uint8_t* paths /* 2n x 48 */,
                             uint8_t* reg_flags, uint8_t* id_flags, uint8_t* body, uint64_t body_cap, uint64_t* body_off /* n+1 */);
int afc_did_reregister_batch_dev(afc_ctx* ctx, const uint8_t* d_master_seed, const uint8_t* server_id, uint64_t server_id_len, const uint8_t* d_agent_cols,
                                 const uint64_t* d_agent_col_off, const uint32_t* d_agent_index, const uint64_t* d_id_idx, const uint8_t* d_ids,
                                 const uint64_t* d_id_off, const uint64_t* d_reg_idx, const uint8_t* d_reg_cols, const uint64_t* d_reg_col_off, uint32_t n,
                                 uint8_t* d_state, uint32_t* d_counts, uint8_t* d_expanded96, uint8_t* d_pks, uint8_t* d_dids, uint8_t* d_paths,
                                 uint8_t* d_reg_flags, uint8_t* d_id_flags, uint8_t* d_body, uint64_t body_cap, uint64_t* d_body_off, void* stream);

/* ---- N4: audit proofs for bulk offline verification (`af vc verify`, internal/cli/vc.go:159-331; export bundles,
 * internal/handlers/ui/did.go:533-865) ------------------------------------------------------------------------
 * afc_merkle_tree materialises every level over a fixed set of leaf hashes (device memory, ~2n x 32 B) so that RFC 6962
 * §2.1.1 audit paths can be read out in bulk; afc_merkle_verify_inclusion_batch checks many paths against one root on
 * the device (RFC 9162 §2.1.3.2).  proof_off: m+1 offsets in units of 32-byte nodes. */
typedef struct afc_merkle_tree afc_merkle_tree;
int afc_merkle_tree_build(afc_ctx* ctx, const uint8_t* leaf_hashes32, uint64_t n, afc_merkle_tree** out);
int afc_merkle_tree_build_dev(afc_ctx* ctx, const uint8_t* d_leaf_hashes32, uint64_t n, afc_merkle_tree** out);
void afc_merkle_tree_free(afc_merkle_tree* t);
int afc_merkle_tree_root(afc_merkle_tree* t, uint8_t root32[32], uint64_t* n_leaves, uint32_t* max_proof_nodes);
int afc_merkle_tree_inclusion_proofs(afc_merkle_tree* t, const uint64_t* indices, uint32_t m, uint8_t* proofs /* m x max_proof_nodes x 32 */,
                                     uint32_t* proof_lens /* m, in nodes */);
int afc_merkle_verify_inclusion_batch(afc_ctx* ctx, const uint8_t* leaf_hashes32, const uint64_t* indices, uint64_t tree_size,
                                      const uint8_t* proofs, const uint32_t* proof_off, const uint8_t root32[32], uint32_t m, uint8_t* ok);
/* RFC 6962 §2.1.2 consistency proof between the first `first` leaves (0 < first <= n) and the whole tree: at most
 * 2 * max_proof_nodes nodes are written to `proof`, their number to *n_nodes.  afc_merkle_verify_consistency_batch checks
 * m earlier checkpoints (first_sizes[i], first_roots32[i]) against one later (second_size, second_root32) on the device
 * (RFC 9162 §2.1.4.2); ok[i] = 0 for first_sizes[i] == 0 or > second_size. */
int afc_merkle_tree_consistency_proof(afc_merkle_tree* t, uint64_t first, uint8_t* proof, uint32_t* n_nodes);
int afc_merkle_verify_consistency_batch(afc_ctx* ctx, const uint64_t* first_sizes, const uint8_t* first_roots32, uint64_t second_size,
                                        const uint8_t second_root32[32], const uint8_t* proofs, const uint32_t* proof_off, uint32_t m, uint8_t* ok);

/* ---- multi-GPU (SURVEY.md §8e): independent shards, one exchange step --------------------------------
 * Each rank appends its contiguous, 2^k-aligned leaf range to its own afc_merkle; the 32-byte subtree
 * roots are all-gathered (NCCL over NVLink) and every rank folds the top levels redundantly.
 * NCCL is dlopen'ed lazily (libnccl.so.2); unique_id is ncclUniqueId (128 bytes). */
int afc_comm_unique_id(uint8_t id128[128]);
int afc_comm_init(afc_ctx* ctx, int nranks, int rank, const uint8_t id128[128]);
int afc_comm_allgather_roots(afc_ctx* ctx, const uint8_t local_root32[32], uint8_t* all_roots /* nranks x 32 */);
int afc_comm_destroy(afc_ctx* ctx);

/* ---- N3: text codecs either side of the kernels (device pointers) ------------------------------------------------------
 * base64.RawURLEncoding of signatures / digests (internal/services/vc_service.go:465,514) and hex.EncodeToString of the
 * webhook tag (internal/services/webhook_dispatcher.go:473) for n fixed-size records of item_bytes each.
 * out: n x ceil(item_bytes*4/3) characters (no padding), resp. n x 2*item_bytes lowercase hex characters. */
int afc_b64url_encode_fixed_dev(afc_ctx* ctx, const uint8_t* d_in, uint32_t item_bytes, uint32_t n, uint8_t* d_out, void* stream);
int afc_hex_encode_fixed_dev(afc_ctx* ctx, const uint8_t* d_in, uint32_t item_bytes, uint32_t n, uint8_t* d_out, void* stream);

/* ---- canonical form on the device (SURVEY.md §8f N3) ---------------------------------------------------------------
 * What the reference signs is json.Marshal of a fixed struct (VCDocument pkg/types/did_types.go:135-220; marshalled at
 * internal/services/vc_service.go:436-439 for signing and :201 for storage; ExecutionWebhookPayload pkg/types/webhook.go:42-53,
 * marshalled at internal/services/webhook_dispatcher.go:286-300): constant text interleaved with a fixed number of values.
 * n documents out[i] = seg[0] || v(i,0) || seg[1] || ... || v(i,F-1) || seg[F]; v(i,f) = d_fields[d_field_off[i*F+f] .. [i*F+f+1])
 * written according to d_kinds[f]: AFC_JSON_STRING = Go encoding/json string escaping (HTML-safe; U+2028/9; invalid UTF-8
 * becomes \ufffd byte by byte) without the quotes — the template supplies them; AFC_JSON_RAW = copied (numbers, pre-rendered
 * optional members).  d_seg_off: F+2 offsets into d_segs.  afc_json_fill_sizes_dev leaves the n+1 output offsets in
 * d_out_off (and, if total_bytes is not NULL, synchronises and returns the total); afc_json_fill_dev writes the bytes. */
#define AFC_JSON_STRING 0
#define AFC_JSON_RAW 1
int afc_json_fill_sizes_dev(afc_ctx* ctx, const uint8_t* d_segs, const uint32_t* d_seg_off, const uint8_t* d_kinds, uint32_t n_fields,
                            const uint8_t* d_fields, const uint64_t* d_field_off, uint32_t n, uint64_t* d_out_off, uint64_t* total_bytes,
                            void* stream);
int afc_json_fill_dev(afc_ctx* ctx, const uint8_t* d_segs, const uint32_t* d_seg_off, const uint8_t* d_kinds, uint32_t n_fields,
                      const uint8_t* d_fields, const uint64_t* d_field_off, uint32_t n, const uint64_t* d_out_off, uint8_t* d_out,
                      void* stream);

/* ---- N2: batching ingest dispatcher (BASELINE.json configs[4]: sustained mixed ingest) ------------------------------
 * One "agent action" = Ed25519 signature over the credential bytes (expanded key `key_index` of the identity cache) +
 * HMAC-SHA256 webhook tag + one audit-log leaf (the signature) appended to an RFC 6962 log owned by the dispatcher.
 * Replaces the reference's one-per-request issuing (internal/handlers/did_handlers.go:192 ->
 * internal/services/vc_service.go:138) and its 4-goroutine webhook worker pool (internal/services/webhook_dispatcher.go:
 * 97-128, 261-320) with GPU batches: flush at `batch_max` actions or after `linger_us`.  Thread-safe; submit blocks only
 * when both staging buffers are full (back-pressure). */
typedef struct afc_ingest afc_ingest;
typedef struct afc_ingest_stats {
    uint64_t submitted, completed, batches;
    double avg_batch;
    uint32_t p50_us, p99_us, max_us;       /* submit -> results-on-host latency */
    uint64_t log_size;
    uint8_t log_root[32];
    int last_error;
} afc_ingest_stats;
int afc_ingest_new(afc_ctx* ctx, const uint8_t* expanded96, uint32_t n_keys, uint32_t batch_max, uint32_t linger_us,
                   uint32_t max_msg, uint32_t max_key, uint32_t max_body, afc_ingest** out);
void afc_ingest_free(afc_ingest* g);
int afc_ingest_submit(afc_ingest* g, uint32_t key_index, const uint8_t* msg, uint32_t msg_len, const uint8_t* hkey, uint32_t hkey_len,
                      const uint8_t* body, uint32_t body_len, uint64_t* ticket);
int afc_ingest_wait(afc_ingest* g, uint64_t ticket, uint8_t sig64[64], uint8_t tag32[32]);
int afc_ingest_flush(afc_ingest* g);
int afc_ingest_stats_get(afc_ingest* g, afc_ingest_stats* out);
/* native open-loop load generator: Poisson arrivals at rate_per_s for `seconds` from `producers` threads (32-byte HMAC keys) */
int afc_ingest_soak(afc_ingest* g, double rate_per_s, double seconds, uint32_t producers, uint32_t msg_len, uint32_t body_len,
                    uint64_t seed, afc_ingest_stats* out, double* achieved_rate, uint64_t* late_submits);

/* ---- diagnostics --------------------------------------------------------------------------------
 * afc_selftest: runs the PTX field arithmetic against the portable reference ON THE DEVICE for `iters`
 * random operands (returns number of mismatches, or negative error).
 * afc_microbench: register-only throughput of a primitive; which = 0 fe_mul, 1 fe_sq, 2 fe_add,
 * 3 sha256 compress, 4 sha512 compress; returns primitive-ops per second (whole GPU) in *ops_per_s. */
int afc_selftest(afc_ctx* ctx, uint32_t iters);
/* afc_staging_find: counts the occurrences of pattern (1..64 bytes) in the context's staging memory — every lane's device slot buffers
 * and pinned bounce buffers — waiting until no host-buffer call is running.  For tests that check that no secret (a master seed, a derived
 * seed, an expanded key) outlives a call. */
int afc_staging_find(afc_ctx* ctx, const uint8_t* pattern, uint32_t len, uint64_t* hits);
/* Per-kernel CUDA-event timing (tracing hook, SURVEY.md §5): between begin and end every kernel this ctx launches is
 * bracketed by two events on its own stream; afc_profile_end synchronises the device and returns one aggregated entry
 * per kernel name (returns the number of entries, or a negative error). */
typedef struct afc_profile_entry {
    char name[48];
    uint32_t count;
    double total_ms, min_ms, max_ms;
} afc_profile_entry;
int afc_profile_begin(afc_ctx* ctx, int max_launches);
int afc_profile_end(afc_ctx* ctx, afc_profile_entry* out, int cap);
int afc_microbench(afc_ctx* ctx, int which, uint32_t iters, double* ops_per_s, double* ms);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* AFCRYPTO_H */
