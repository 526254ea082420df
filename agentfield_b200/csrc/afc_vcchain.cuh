// Workflow VC chains served on the device (afc_vc_workflow_chain_batch, include/afcrypto.h): the body gin's c.JSON writes for
// types.WorkflowVCChainResponse (pkg/types/did_types.go:287-295) after GetWorkflowVCChain (internal/services/vc_service.go:292-338).
//
//   vcc_time_ok / vcc_put_time   time.Time.MarshalJSON (RFC3339Nano: fraction with trailing zeros trimmed, Z or ±hh:mm) of Unix seconds,
//                                nanoseconds and a UTC offset; declined (the workflow goes to the host) for an offset that is not a whole
//                                number of minutes or is 24 hours or more, and a local year outside 1..9999.
//   vcc_compact                  appendCompact(dst, src, escapeHTML = true) of a vc_document jv_validate accepted: whitespace outside
//                                strings dropped, < > & U+2028 U+2029 escaped, every other byte copied.
//   vcc_record                   one ExecutionVC record in struct order (agent_node_id / workflow_name omitted when nil, vc_document null
//                                when nil; parent_vc_id and child_vc_ids are never set by storage, vc_storage.go:234-263, so never written).
//   vcc_did_wanted / vcc_method  collectDIDResolutionBundle's filter (:810-870: "", "did:key:", and what strings.TrimSpace empties) and
//                                strings.Split(did, ":")[1].
//   vcc_entry                    one bundle member: the DID as a Go-escaped key and its DIDResolutionEntry, public_key_jwk being
//                                ed25519PublicKeyToJWK's text of the directory's key.
//   vcc_frame                    the text of the response around the regions other threads write: the records, the workflow credential's
//                                component ids, its stored document and the bundle's members.
//
// Shared by the kernels of k_vcchain.cu and the CPU build of the same logic in tests/hostsim.
#pragma once
#include "afc_didreg.cuh"
#include "afc_jsonval.cuh"
#include "afc_vcworkflow.cuh"

namespace afc {

enum {
    VCC_COLUMNS = 2,          // workflow_vc_id, resolved_at (AFC_CHAIN_WORKFLOW_COLUMNS)
    VCC_COL_WF_VC_ID = 0, VCC_COL_RESOLVED_AT = 1,
    VCC_REC_COLUMNS = 13,     // AFC_CHAIN_RECORD_COLUMNS
    VCC_R_EXECUTION = 0, VCC_R_WORKFLOW = 1, VCC_R_SESSION = 2, VCC_R_AGENT = 3, VCC_R_WF_NAME = 4, VCC_R_ISSUER = 5, VCC_R_TARGET = 6,
    VCC_R_CALLER = 7, VCC_R_DOC = 8, VCC_R_SIGNATURE = 9, VCC_R_URI = 10, VCC_R_INPUT = 11, VCC_R_OUTPUT = 12,
    VCC_AGENT_NIL = 1, VCC_NAME_NIL = 2, VCC_DOC_NIL = 4,          // AFC_CHAIN_*_NIL record flags
    VCC_TIME_CHARS = 35,      // 2006-01-02T15:04:05.999999999-07:00
    VCC_RESOLVED_MAX = 64,    // longer resolved_at columns are declined (the reference writes 20 characters)
    VCC_DID_MAX = 128,        // a workflow whose bundle would hold a longer DID is declined (the registry's did:key DIDs have 55)
};
enum : uint32_t { VCC_BUILT = 0, VCC_HOST = 1 };                 // AFC_CHAIN_BUILT / _HOST
constexpr uint32_t VCC_NONE = 0xffffffffu;                       // a DID occurrence the bundle does not take

// ---- time.Time.MarshalJSON

AFC_HD bool vcc_time_ok(int64_t sec, int64_t nsec, int64_t off) {
    if (nsec < 0 || nsec >= 1000000000LL || off % 60 != 0 || off <= -86400 || off >= 86400) return false;
    if (sec < VCW_SEC_MIN - 86400 || sec > VCW_SEC_MAX + 86400) return false;     // keeps sec + off from overflowing
    const int64_t local = sec + off;
    return local >= VCW_SEC_MIN && local <= VCW_SEC_MAX;
}
template <class Sink>
AFC_HD void vcc_put_time(Sink& out, int64_t sec, int64_t nsec, int64_t off) {
    vcw_put_civil(out, sec + off);
    if (nsec) {
        out.put('.');
        uint32_t v = (uint32_t)nsec, digits = 9;
        while (v % 10 == 0) { v /= 10; --digits; }
        uint32_t p = 1;
        for (uint32_t k = 1; k < digits; k++) p *= 10;
        for (; p; p /= 10) out.put('0' + v / p % 10);
    }
    if (off == 0) { out.put('Z'); return; }
    const uint32_t a = (uint32_t)(off < 0 ? -off : off) / 60;
    out.put(off < 0 ? '-' : '+');
    vcw_put2(out, a / 60); out.put(':'); vcw_put2(out, a % 60);
}

// ---- json.RawMessage

// appendCompact with escapeHTML of a text jv_validate accepted (so every quote and backslash is where the grammar puts it)
template <class Sink>
AFC_HD void vcc_compact(Sink& out, const uint8_t* d, uint64_t len) {
    bool in_str = false, esc = false;
    for (uint64_t i = 0; i < len; i++) {
        const uint32_t c = d[i];
        if (!in_str) {
            if (c == ' ' || c == '\t' || c == '\n' || c == '\r') continue;
            if (c == '"') in_str = true;
            out.put(c);
        } else if (esc) {
            esc = false;
            out.put(c);
        } else if (c == '\\') {
            esc = true;
            out.put(c);
        } else if (c == '"') {
            in_str = false;
            out.put(c);
        } else if (c == '<' || c == '>' || c == '&') {
            out.put('\\'); out.put('u'); out.put('0'); out.put('0'); out.put(json_hex_digit(c >> 4)); out.put(json_hex_digit(c & 15));
        } else if (c == 0xE2 && i + 2 < len && d[i + 1] == 0x80 && (d[i + 2] & ~1u) == 0xA8) {
            out.put('\\'); out.put('u'); out.put('2'); out.put('0'); out.put('2'); out.put(json_hex_digit(d[i + 2] & 15));
            i += 2;
        } else {
            out.put(c);
        }
    }
}

// ---- one ExecutionVC record

struct VccStr { const uint8_t* p; uint64_t len; };
struct VccRecord {
    VccStr vc_id, status;                 // the issue call's two record columns
    const uint8_t* cols;                  // the chain's: column c is cols[coff[c] .. coff[c + 1])
    const uint64_t* coff;
    uint32_t flags;
    int64_t doc_size, sec, nsec, zone;    // zone: created_at's UTC offset in seconds
    AFC_HDM VccStr col(uint32_t c) const { VccStr s; s.p = cols + coff[c]; s.len = coff[c + 1] - coff[c]; return s; }
};

// VCC_HOST when json.Marshal of the record fails here or is not written by this code: a non-nil document that is empty or not JSON (or
// that jv_validate leaves to the host), a created_at MarshalJSON would not write as vcc_put_time does
AFC_HD uint32_t vcc_record_state(const VccRecord& r) {
    if (!vcc_time_ok(r.sec, r.nsec, r.zone)) return VCC_HOST;
    if (!(r.flags & VCC_DOC_NIL) && jv_validate(r.col(VCC_R_DOC).p, r.col(VCC_R_DOC).len) != JV_OK) return VCC_HOST;
    return VCC_BUILT;
}

template <class Sink>
AFC_HD void vcc_str(Sink& out, const char* name, VccStr s) {
    vci_put_text(out, name);
    go_json_escape(out, s.p, s.len);
    out.put('"');
}
template <class Sink>
AFC_HD void vcc_record(Sink& out, const VccRecord& r) {
    vcc_str(out, "{\"vc_id\":\"", r.vc_id);
    vcc_str(out, ",\"execution_id\":\"", r.col(VCC_R_EXECUTION));
    vcc_str(out, ",\"workflow_id\":\"", r.col(VCC_R_WORKFLOW));
    vcc_str(out, ",\"session_id\":\"", r.col(VCC_R_SESSION));
    if (!(r.flags & VCC_AGENT_NIL)) vcc_str(out, ",\"agent_node_id\":\"", r.col(VCC_R_AGENT));
    if (!(r.flags & VCC_NAME_NIL)) vcc_str(out, ",\"workflow_name\":\"", r.col(VCC_R_WF_NAME));
    vcc_str(out, ",\"issuer_did\":\"", r.col(VCC_R_ISSUER));
    vcc_str(out, ",\"target_did\":\"", r.col(VCC_R_TARGET));
    vcc_str(out, ",\"caller_did\":\"", r.col(VCC_R_CALLER));
    vci_put_text(out, ",\"vc_document\":");
    if (r.flags & VCC_DOC_NIL) vci_put_text(out, "null");
    else vcc_compact(out, r.col(VCC_R_DOC).p, r.col(VCC_R_DOC).len);
    vcc_str(out, ",\"signature\":\"", r.col(VCC_R_SIGNATURE));
    vcc_str(out, ",\"storage_uri\":\"", r.col(VCC_R_URI));
    vci_put_text(out, ",\"document_size_bytes\":");
    vci_put_int(out, r.doc_size);
    vcc_str(out, ",\"input_hash\":\"", r.col(VCC_R_INPUT));
    vcc_str(out, ",\"output_hash\":\"", r.col(VCC_R_OUTPUT));
    vcc_str(out, ",\"status\":\"", r.status);
    vci_put_text(out, ",\"created_at\":\"");
    vcc_put_time(out, r.sec, r.nsec, r.zone);
    vci_put_text(out, "\"}");
}

// ---- the DID resolution bundle

// unicode.IsSpace of the rune at d[i] (valid UTF-8 only; an invalid byte is utf8.RuneError, not a space): its length, or 0
AFC_HD uint32_t vcc_space_len(const uint8_t* d, uint64_t i, uint64_t len) {
    const uint32_t b = d[i];
    if (b == ' ' || (b >= '\t' && b <= '\r')) return 1;
    const uint32_t b1 = i + 1 < len ? d[i + 1] : 0, b2 = i + 2 < len ? d[i + 2] : 0;
    if (b == 0xC2 && (b1 == 0x85 || b1 == 0xA0)) return 2;                                       // U+0085 U+00A0
    if (b == 0xE1 && b1 == 0x9A && b2 == 0x80) return 3;                                          // U+1680
    if (b == 0xE2 && b1 == 0x80 && ((b2 >= 0x80 && b2 <= 0x8A) || b2 == 0xA8 || b2 == 0xA9 || b2 == 0xAF)) return 3;   // U+2000-200A 2028 2029 202F
    if (b == 0xE2 && b1 == 0x81 && b2 == 0x9F) return 3;                                          // U+205F
    if (b == 0xE3 && b1 == 0x80 && b2 == 0x80) return 3;                                          // U+3000
    return 0;
}
// the bundle looks the DID up: not "", not "did:key:", not all white space
AFC_HD bool vcc_did_wanted(const uint8_t* d, uint64_t len) {
    if (len == 0) return false;
    if (len == 8 && d[0] == 'd' && d[1] == 'i' && d[2] == 'd' && d[3] == ':' && d[4] == 'k' && d[5] == 'e' && d[6] == 'y' && d[7] == ':') return false;
    for (uint64_t i = 0; i < len;) {
        const uint32_t k = vcc_space_len(d, i, len);
        if (!k) return true;
        i += k;
    }
    return false;
}
// the DID's method: strings.Split(did, ":")[1] for a did: prefix and more, else "key" (returned as a null p)
AFC_HD VccStr vcc_method(const uint8_t* d, uint64_t len) {
    VccStr m; m.p = nullptr; m.len = 0;
    if (len <= 4 || !(d[0] == 'd' && d[1] == 'i' && d[2] == 'd' && d[3] == ':')) return m;
    uint64_t e = 4;
    while (e < len && d[e] != ':') ++e;
    m.p = d + 4; m.len = e - 4;
    return m;
}
// "did":{"method":...,"public_key_jwk":{...},"resolved_from":"bundled","resolved_at":...}; pk: the key as little-endian words
template <class Sink>
AFC_HD void vcc_entry(Sink& out, VccStr did, const uint32_t pk[8], VccStr resolved_at) {
    out.put('"');
    go_json_escape(out, did.p, did.len);
    vci_put_text(out, "\":{\"method\":\"");
    const VccStr m = vcc_method(did.p, did.len);
    if (m.p) go_json_escape(out, m.p, m.len);
    else vci_put_text(out, "key");
    vci_put_text(out, "\",\"public_key_jwk\":{\"alg\":\"EdDSA\",\"crv\":\"Ed25519\",\"kty\":\"OKP\",\"use\":\"sig\",\"x\":\"");
    didr_b64_32(out, pk);
    vcc_str(out, "\"},\"resolved_from\":\"bundled\",\"resolved_at\":\"", resolved_at);
    out.put('}');
}

// ---- the response around the regions

struct VccFrame {
    VccStr workflow_id, session_id, issuer, wf_vc_id;
    uint32_t status, cnt, completed;
    int64_t start[3], end[3], snap[3];    // (seconds, nanoseconds, UTC offset)
    bool has_end, has_bundle;
    const uint8_t* proof_value;           // 86 characters
    uint64_t doc_len;
};
enum { VCC_PARTS = 5 };
// Part k of the frame: 0 before the records, 1 before the credential's component ids (ending with its '['), 2 from the ']' after them to
// the stored document, 3 after it to the bundle's members, 4 the end
template <class Sink>
AFC_HD void vcc_frame(Sink& out, const VccFrame& f, uint32_t part) {
    switch (part) {
    case 0:
        vcc_str(out, "{\"workflow_id\":\"", f.workflow_id);
        vci_put_text(out, ",\"component_vcs\":[");
        break;
    case 1:
        vcc_str(out, "],\"workflow_vc\":{\"workflow_id\":\"", f.workflow_id);
        vcc_str(out, ",\"session_id\":\"", f.session_id);
        vci_put_text(out, ",\"component_vcs\":[");
        break;
    case 2:
        vcc_str(out, "],\"workflow_vc_id\":\"", f.wf_vc_id);
        vci_put_text(out, ",\"status\":\"");
        vcw_put_status(out, f.status);
        vci_put_text(out, "\",\"start_time\":\"");
        vcc_put_time(out, f.start[0], f.start[1], f.start[2]);
        if (f.has_end) {
            vci_put_text(out, "\",\"end_time\":\"");
            vcc_put_time(out, f.end[0], f.end[1], f.end[2]);
        }
        vci_put_text(out, "\",\"total_steps\":");
        vci_put_int(out, f.cnt);
        vci_put_text(out, ",\"completed_steps\":");
        vci_put_int(out, f.completed);
        vci_put_text(out, ",\"vc_document\":");
        break;
    case 3:
        vci_put_text(out, ",\"signature\":\"");
        for (uint32_t k = 0; k < VCI_PV_CHARS; k++) out.put(f.proof_value[k]);
        out.put('"');
        if (f.issuer.len) vcc_str(out, ",\"issuer_did\":\"", f.issuer);
        vci_put_text(out, ",\"snapshot_time\":\"");
        vcc_put_time(out, f.snap[0], f.snap[1], f.snap[2]);
        vci_put_text(out, "\",\"storage_uri\":\"\",\"document_size_bytes\":");
        vci_put_int(out, (int64_t)f.doc_len);
        vci_put_text(out, "},\"total_steps\":");
        vci_put_int(out, f.cnt);
        vci_put_text(out, ",\"status\":\"");
        vcw_put_status(out, f.status);
        out.put('"');
        if (f.has_bundle) vci_put_text(out, ",\"did_resolution_bundle\":{");
        break;
    default:
        if (f.has_bundle) out.put('}');
        out.put('}');
        break;
    }
}

// The constant text the bound allows per workflow, per record and per DID occurrence (a member's key and method are at most 6 bytes per
// byte of a DID of at most VCC_DID_MAX bytes), besides 6 bytes per escaped column byte
constexpr uint64_t VCC_FRAME_FIXED = 520 + 3 * VCC_TIME_CHARS + 4 * 20 + VCI_PV_CHARS;
constexpr uint64_t VCC_RECORD_FIXED = 300 + VCC_TIME_CHARS + 20;
constexpr uint64_t VCC_ENTRY_FIXED = 160 + 43 + 6 * VCC_RESOLVED_MAX + 12 * VCC_DID_MAX;

}  // namespace afc
