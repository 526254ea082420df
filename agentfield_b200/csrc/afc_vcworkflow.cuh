// Workflow credentials issued on the device (afc_vc_issue_workflow_batch, include/afcrypto.h): what generateWorkflowVCDocument
// (internal/services/vc_service.go:525-632) computes and stores for one workflow and its ExecutionVC records.
//
//   vcw_record_class   NormalizeExecutionStatus of one record (vc_status_class on a column: decided for printable ASCII and \t \n \v \f \r
//                      only) and whether its created_at is one RFC 3339 formats in four digits (0001-01-01T00:00:00Z ..
//                      9999-12-31T23:59:59Z, nanoseconds in [0, 10^9)); anything else makes the workflow VCW_HOST.
//   vcw_reduce         determineWorkflowStatus (:721-772), countCompletedSteps (:775-787) and the start / end loop (:546-563): the
//                      first record with the earliest time (strict Before) and the first with the latest (strict After).
//   vcw_doc_sizes / vcw_doc_fill  createWorkflowVCDocument + json.Marshal (:635-683, signWorkflowVC :686-693 for the signing form, :611 for the stored
//                      form): the constant text of types.WorkflowVCDocument interleaved with the workflow's columns, Go-escaped, all but
//                      the ids inside the componentVcIds array: each record writes its own id there (vcw_put_id), in both forms, since the
//                      prefix through "proof": is common to them.
//   vcw_put_time       time.Time.UTC().Format(time.RFC3339) of Unix seconds: integer civil-from-days arithmetic, 20 characters (vcw_put_civil
//                      writes the first 19, which the chain call's RFC3339Nano writer shares).
//
// Deliberate deviation: a workflow with no records starts at time.Now() in the reference (:563), read a second time for snapshotTime.  Here
// its startTime is the snapshot_time column's text, as the host mirror (services.generate_workflow_vc_batch) writes it.
//
// Shared by the kernels of k_vcworkflow.cu and the CPU build of the same logic in tests/hostsim.
#pragma once
#include "afc_vcdoc.cuh"
#include "afc_vcissue.cuh"

namespace afc {

enum {
    VCW_COLUMNS = 7,         // workflow_id, session_id, issuer_did, vc_id, issuance_date, snapshot_time, proof_created (AFC_WORKFLOW_COLUMNS)
    VCW_COL_WORKFLOW = 0, VCW_COL_SESSION = 1, VCW_COL_ISSUER = 2, VCW_COL_VC_ID = 3, VCW_COL_ISSUANCE = 4, VCW_COL_SNAPSHOT = 5,
    VCW_COL_PROOF_CREATED = 6,
    VCW_REC_COLUMNS = 2,     // vc_id, status of each record (AFC_WORKFLOW_RECORD_COLUMNS)
    VCW_TIME_CHARS = 20,     // 2006-01-02T15:04:05Z
};
enum : uint32_t { VCW_BUILT = 0, VCW_HOST = 1 };                  // AFC_WORKFLOW_BUILT / _HOST
constexpr uint32_t VCW_NONE = 0xffffffffu;                        // summary[2] / [3]: no such record
constexpr int64_t VCW_SEC_MIN = -62135596800LL;                   // 0001-01-01T00:00:00Z
constexpr int64_t VCW_SEC_MAX = 253402300799LL;                   // 9999-12-31T23:59:59Z
constexpr uint32_t VCW_R_HOST = 8;                                // record class: bits 0-2 the status id, this bit = the workflow goes to the host

// What follows each literal of the program
enum : uint8_t {
    VCW_V_NONE = 0x80, VCW_V_IDS, VCW_V_COUNT, VCW_V_STATUS, VCW_V_START, VCW_V_END, VCW_V_PROOF_VALUE,
    // values below 0x80 are column indices (escaped as Go strings)
};

// The constant text and column map of json.Marshal(types.WorkflowVCDocument), staged once per block in shared memory.  Piece VCW_P_IDS
// ends the head (its value is the componentVcIds array); pieces (VCW_P_IDS, VCW_COMMON) run to "proof":; piece VCW_SIGN_TAIL is the
// zero-valued proof the reference signs over; pieces (VCW_SIGN_TAIL, VCW_PIECES) are the stored proof.
enum { VCW_P_IDS = 5, VCW_COMMON = 16, VCW_SIGN_TAIL = 16, VCW_PIECES = 21, VCW_POOL_WORDS = 256 };
struct VcwProgram {
    uint32_t pool[VCW_POOL_WORDS];
    uint16_t lit_off[VCW_PIECES], lit_len[VCW_PIECES];
    uint8_t val[VCW_PIECES];
};

// Builds the program (host code); returns the bytes of literal text (0 if the pool is too small, which would be a bug)
static inline uint32_t vcw_program_build(VcwProgram* P) {
    static const struct { const char* lit; uint8_t val; } pieces[VCW_PIECES] = {
        {"{\"@context\":[\"https://www.w3.org/2018/credentials/v1\",\"https://agentfield.example.com/contexts/workflow/v1\"],"
         "\"type\":[\"VerifiableCredential\",\"AgentFieldWorkflowCredential\"],\"id\":\"urn:agentfield:workflow-vc:", VCW_COL_VC_ID},
        {"\",\"issuer\":\"", VCW_COL_ISSUER},
        {"\",\"issuanceDate\":\"", VCW_COL_ISSUANCE},
        {"\",\"credentialSubject\":{\"workflowId\":\"", VCW_COL_WORKFLOW},
        {"\",\"sessionId\":\"", VCW_COL_SESSION},
        {"\",\"componentVcIds\":", VCW_V_IDS},
        {",\"totalSteps\":", VCW_V_COUNT},
        {",\"completedSteps\":", VCW_V_COUNT},
        {",\"status\":\"", VCW_V_STATUS},
        {"\",\"startTime\":\"", VCW_V_START},
        {"\"", VCW_V_END},
        {",\"snapshotTime\":\"", VCW_COL_SNAPSHOT},
        {"\",\"orchestrator\":{\"did\":\"", VCW_COL_ISSUER},
        {"\",\"type\":\"agentfield_server\",\"agentNodeDid\":\"", VCW_COL_ISSUER},
        {"\"},\"audit\":{\"inputDataHash\":\"\",\"outputDataHash\":\"\",\"metadata\":{\"agentfield_version\":\"1.0.0\",\"total_executions\":",
         VCW_V_COUNT},
        {",\"vc_version\":\"1.0\",\"workflow_type\":\"agent_execution_chain\"}}},\"proof\":", VCW_V_NONE},
        {"{\"type\":\"\",\"created\":\"\",\"verificationMethod\":\"\",\"proofPurpose\":\"\",\"proofValue\":\"\"}}", VCW_V_NONE},
        {"{\"type\":\"Ed25519Signature2020\",\"created\":\"", VCW_COL_PROOF_CREATED},
        {"\",\"verificationMethod\":\"", VCW_COL_ISSUER},
        {"#key-1\",\"proofPurpose\":\"assertionMethod\",\"proofValue\":\"", VCW_V_PROOF_VALUE},
        {"\"}}", VCW_V_NONE},
    };
    memset(P, 0, sizeof *P);
    uint8_t* pool = (uint8_t*)P->pool;
    uint32_t at = 0, text = 0;
    for (int k = 0; k < VCW_PIECES; k++) {
        const uint32_t len = (uint32_t)strlen(pieces[k].lit);
        if (at + len > sizeof P->pool) return 0;
        memcpy(pool + at, pieces[k].lit, len);
        P->lit_off[k] = (uint16_t)at; P->lit_len[k] = (uint16_t)len; P->val[k] = pieces[k].val;
        at = (at + len + 3) & ~3u;
        text += len;
    }
    return text;
}

// ---- one record

// The record's class: its status id (0 unknown ... 7 timeout), | VCW_R_HOST when the workflow cannot be built here
AFC_HD uint32_t vcw_record_class(const uint8_t* status, uint64_t status_len, int64_t sec, int64_t nsec) {
    const uint32_t c = vc_status_class(status, status_len, false);
    const bool host = c == VC_UNDECIDED || sec < VCW_SEC_MIN || sec > VCW_SEC_MAX || nsec < 0 || nsec >= 1000000000LL;
    return host ? VCW_R_HOST : c;
}

// The bytes one record adds to the componentVcIds array: its escaped id in quotes (the comma before every id but the first is counted
// by the workflow)
AFC_HD uint64_t vcw_id_bytes(const uint8_t* id, uint64_t len) {
    ByteCounter c; c.init();
    go_json_escape(c, id, len);
    return c.n + 2;
}

// ---- one workflow

struct VcwPlan {
    uint32_t state;          // VCW_BUILT / VCW_HOST
    uint32_t status;         // vc_status_id numbering
    uint32_t completed;      // records that normalise to succeeded
    uint32_t start, end;     // record indices relative to the workflow's first, VCW_NONE if none (end: also when the status is not terminal)
    uint64_t ids_bytes;      // the componentVcIds array, brackets included
};

AFC_HD bool vcw_time_before(int64_t s0, int64_t n0, int64_t s1, int64_t n1) { return s0 < s1 || (s0 == s1 && n0 < n1); }

// determineWorkflowStatus's precedence over the set of normalised statuses seen (bit k = status id k); no records is pending
AFC_HD uint32_t vcw_status_of(uint32_t seen, uint32_t cnt) {
    if (cnt == 0) return 1;
    if (seen & (1u << 5)) return 5;                               // failed
    if (seen & (1u << 7)) return 7;                               // timeout
    if (seen & (1u << 6)) return 6;                               // cancelled
    if (seen & (1u << 3)) return 3;                               // running
    if (seen & (1u << 2)) return 2;                               // queued
    if (seen & (1u << 1)) return 1;                               // pending
    if (seen & 1u) return 0;                                      // unknown
    return 4;                                                     // every record succeeded
}

// cls, id_len: the workflow's cnt records' classes and vcw_id_bytes; created: their (seconds, nanoseconds) pairs
AFC_HD VcwPlan vcw_reduce(const uint8_t* cls, const uint64_t* id_len, const int64_t* created, uint32_t cnt) {
    VcwPlan p;
    uint32_t seen = 0, host = 0, done = 0, lo = 0, hi = 0;
    uint64_t ids = 2 + (cnt ? cnt - 1 : 0);
    for (uint32_t k = 0; k < cnt; k++) {
        const uint32_t c = cls[k];
        host |= c & VCW_R_HOST;
        seen |= 1u << (c & 7u);
        done += (c & 7u) == 4;
        ids += id_len[k];
        if (vcw_time_before(created[2 * k], created[2 * k + 1], created[2 * lo], created[2 * lo + 1])) lo = k;
        if (vcw_time_before(created[2 * hi], created[2 * hi + 1], created[2 * k], created[2 * k + 1])) hi = k;
    }
    if (host) { p.state = VCW_HOST; p.status = 0; p.completed = 0; p.start = p.end = 0; p.ids_bytes = 0; return p; }
    p.state = VCW_BUILT;
    p.status = vcw_status_of(seen, cnt);
    p.completed = done;
    p.start = cnt ? lo : VCW_NONE;
    p.end = cnt && p.status >= 4 ? hi : VCW_NONE;                 // IsTerminalExecutionStatus: succeeded, failed, cancelled, timeout
    p.ids_bytes = ids;
    return p;
}

// What the document's text needs of one workflow
struct VcwItem {
    const uint8_t* cols;
    const uint64_t* coff;    // its VCW_COLUMNS + 1 absolute offsets into cols
    uint32_t cnt, status;
    int64_t start_sec, end_sec;
    bool has_end;
    uint64_t ids_bytes;
};

// Two decimal digits, and time.Time.UTC().Format(time.RFC3339) of Unix seconds in [VCW_SEC_MIN, VCW_SEC_MAX]
template <class Sink>
AFC_HD void vcw_put2(Sink& out, uint32_t v) { out.put('0' + v / 10); out.put('0' + v % 10); }
// The civil date and time of Unix seconds without a zone designator: 2006-01-02T15:04:05 (19 characters)
template <class Sink>
AFC_HD void vcw_put_civil(Sink& out, int64_t sec) {
    const int64_t days = (sec >= 0 ? sec : sec - 86399) / 86400;  // floor division
    const uint32_t sod = (uint32_t)(sec - days * 86400);
    // civil from days (proleptic Gregorian, eras of 400 years = 146097 days from 0000-03-01)
    const int64_t z = days + 719468;
    const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
    const uint32_t doe = (uint32_t)(z - era * 146097);
    const uint32_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const uint32_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const uint32_t mp = (5 * doy + 2) / 153;
    const uint32_t d = doy - (153 * mp + 2) / 5 + 1, m = mp < 10 ? mp + 3 : mp - 9;
    const uint32_t y = (uint32_t)(yoe + era * 400 + (m <= 2));
    vcw_put2(out, y / 100); vcw_put2(out, y % 100); out.put('-'); vcw_put2(out, m); out.put('-'); vcw_put2(out, d);
    out.put('T'); vcw_put2(out, sod / 3600); out.put(':'); vcw_put2(out, sod / 60 % 60); out.put(':'); vcw_put2(out, sod % 60);
}
template <class Sink>
AFC_HD void vcw_put_time(Sink& out, int64_t sec) {
    vcw_put_civil(out, sec);
    out.put('Z');
}

template <class Sink>
AFC_HD void vcw_put_status(Sink& out, uint32_t s) {
    switch (s) {
    case 1: vci_put_text(out, "pending"); break;
    case 2: vci_put_text(out, "queued"); break;
    case 3: vci_put_text(out, "running"); break;
    case 4: vci_put_text(out, "succeeded"); break;
    case 5: vci_put_text(out, "failed"); break;
    case 6: vci_put_text(out, "cancelled"); break;
    case 7: vci_put_text(out, "timeout"); break;
    default: vci_put_text(out, "unknown"); break;
    }
}

template <class Sink>
AFC_HD void vcw_col(Sink& out, const VcwItem& it, uint32_t c) { go_json_escape(out, it.cols + it.coff[c], it.coff[c + 1] - it.coff[c]); }

// Every value but the componentVcIds array, which the head / tail split leaves to the records
template <class Sink>
AFC_HD void vcw_value(Sink& out, uint32_t v, const VcwItem& it) {
    if (v < VCW_COLUMNS) { vcw_col(out, it, v); return; }
    switch (v) {
    case VCW_V_COUNT: vci_put_int(out, (int64_t)it.cnt); break;
    case VCW_V_STATUS: vcw_put_status(out, it.status); break;
    case VCW_V_START:
        if (it.cnt) vcw_put_time(out, it.start_sec);
        else vcw_col(out, it, VCW_COL_SNAPSHOT);
        break;
    case VCW_V_END:                                               // *string, omitempty
        if (!it.has_end) break;
        vci_put_text(out, ",\"endTime\":\"");
        vcw_put_time(out, it.end_sec);
        out.put('"');
        break;
    case VCW_V_PROOF_VALUE:                                       // placeholder until the signature exists (vci_proof_one)
        for (uint32_t k = 0; k < VCI_PV_CHARS / 4; k++) out.put4(0x41414141u);
        out.put('A'); out.put('A');
        break;
    default: break;
    }
}

template <class Sink>
AFC_HD void vcw_pieces(Sink& out, const VcwProgram& P, uint32_t k0, uint32_t k1, const VcwItem& it) {
    for (uint32_t k = k0; k < k1; k++) {
        vci_put_lit(out, P.pool, P.lit_off[k], P.lit_len[k]);
        if (k != VCW_P_IDS) vcw_value(out, P.val[k], it);
    }
}

// Both lengths of one workflow's credential, and where its componentVcIds array starts (the same place in both)
AFC_HD void vcw_doc_sizes(const VcwProgram& P, const VcwItem& it, uint64_t* msg_len, uint64_t* doc_len, uint64_t* arr_at) {
    ByteCounter c; c.init();
    vcw_pieces(c, P, 0, VCW_P_IDS + 1, it);
    *arr_at = c.n;
    c.n += it.ids_bytes;
    vcw_pieces(c, P, VCW_P_IDS + 1, VCW_COMMON, it);
    *msg_len = c.n + P.lit_len[VCW_SIGN_TAIL];
    vcw_pieces(c, P, VCW_SIGN_TAIL + 1, VCW_PIECES, it);
    *doc_len = c.n;
}

// Writes the signing message at msg and the stored document (proofValue still a placeholder) at doc, all but the ids between the brackets
AFC_HD void vcw_doc_fill(const VcwProgram& P, const VcwItem& it, uint64_t arr_at, uint8_t* msg, uint8_t* doc) {
    {
        TeeWriter h; h.a.init(msg); h.b.init(doc);
        vcw_pieces(h, P, 0, VCW_P_IDS + 1, it);
        h.put('[');
        h.a.finish(); h.b.finish();
    }
    const uint64_t close = arr_at + it.ids_bytes - 1;
    TeeWriter t; t.a.init(msg + close); t.b.init(doc + close);
    t.put(']');
    vcw_pieces(t, P, VCW_P_IDS + 1, VCW_COMMON, it);
    vcw_pieces(t.a, P, VCW_SIGN_TAIL, VCW_SIGN_TAIL + 1, it);
    t.a.finish();
    vcw_pieces(t.b, P, VCW_SIGN_TAIL + 1, VCW_PIECES, it);
    t.b.finish();
}

// Record k of a workflow writes  "id"  (k == 0) or  ,"id"  at msg / doc, which point at the byte after the array's '[' plus the escaped ids
// and commas of the records before it
AFC_HD void vcw_put_id(const uint8_t* id, uint64_t len, uint32_t k, uint8_t* msg, uint8_t* doc) {
    TeeWriter t; t.a.init(msg); t.b.init(doc);
    if (k) t.put(',');
    t.put('"');
    go_json_escape(t, id, len);
    t.put('"');
    t.a.finish(); t.b.finish();
}
// Where record k's text starts, relative to the array's '[': before = the vcw_id_bytes of the records before it
AFC_HD uint64_t vcw_id_at(uint64_t before, uint32_t k) { return 1 + before + (k ? k - 1 : 0); }

}  // namespace afc
