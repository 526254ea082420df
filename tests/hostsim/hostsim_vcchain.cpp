// TEST-ONLY CPU build of the workflow-chain routines (agentfield_b200/csrc/afc_vcchain.cuh): what the threads of k_vcc_records,
// k_vcc_distinct, k_vcc_sizes and the emit passes do for one workflow, after the workflow-credential passes (afc_vcworkflow.cuh, its
// proofValue a placeholder).  The directory probe and the distinct-rank sort are plain std containers here.  Compiled on its own by
// tests/test_vcchain_hostsim.py.
#define AFC_HOSTSIM 1
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../agentfield_b200/csrc/afc_vcchain.cuh"

using namespace afc;

extern "C" {

// One workflow: its 7 issue columns (8 absolute offsets), its cnt records' issue columns (2 cnt + 1 offsets) and (seconds, nanoseconds),
// its 2 chain columns (3 offsets) and clock, its records' 13 chain columns (13 cnt + 1 offsets), flags, sizes and zones; the directory's
// dir_n DIDs (dir_n + 1 offsets) and keys.  Writes *state and *body_len and, when body is given (body_len plus 32 bytes), the body.
int hs_vcc_chain(const uint8_t* cols, const uint64_t* coff, const uint8_t* rec_cols, const uint64_t* rec_coff, const int64_t* created, uint32_t cnt,
                 const uint8_t* chain_cols, const uint64_t* chain_coff, const int64_t* clock, const uint8_t* crec_cols, const uint64_t* crec_coff,
                 const uint8_t* flags, const int64_t* doc_size, const int32_t* zone, const uint8_t* dir_dids, const uint64_t* dir_off,
                 const uint8_t* dir_pks, uint32_t dir_n, uint32_t* state, uint8_t* body, uint64_t* body_len) {
    static VcwProgram P;
    static bool built = false;
    if (!built) { if (!vcw_program_build(&P)) return -1; built = true; }
    *body_len = 0;
    // the workflow credential, as hs_vcw_issue computes it
    std::vector<uint8_t> cls(cnt + 1);
    std::vector<uint64_t> id_len(cnt + 1);
    for (uint32_t k = 0; k < cnt; k++) {
        const uint64_t a = rec_coff[2 * k], b = rec_coff[2 * k + 1], c = rec_coff[2 * k + 2];
        cls[k] = (uint8_t)vcw_record_class(rec_cols + b, c - b, created[2 * k], created[2 * k + 1]);
        id_len[k] = vcw_id_bytes(rec_cols + a, b - a);
    }
    const VcwPlan p = vcw_reduce(cls.data(), id_len.data(), created, cnt);
    if (p.state == VCW_HOST) { *state = VCC_HOST; return 0; }
    VcwItem it;
    it.cols = cols; it.coff = coff; it.cnt = cnt; it.status = p.status;
    it.start_sec = p.start != VCW_NONE ? created[2 * p.start] : 0;
    it.has_end = p.end != VCW_NONE;
    it.end_sec = it.has_end ? created[2 * p.end] : 0;
    it.ids_bytes = p.ids_bytes;
    uint64_t msg_len, doc_len, arr_at;
    vcw_doc_sizes(P, it, &msg_len, &doc_len, &arr_at);
    std::vector<uint8_t> msg(msg_len + 32), doc(doc_len + 32);
    vcw_doc_fill(P, it, arr_at, msg.data(), doc.data());
    {
        uint64_t before = 0;
        for (uint32_t k = 0; k < cnt; k++) {
            const uint64_t at = arr_at + vcw_id_at(before, k);
            vcw_put_id(rec_cols + rec_coff[2 * k], rec_coff[2 * k + 1] - rec_coff[2 * k], k, msg.data() + at, doc.data() + at);
            before += id_len[k];
        }
    }
    std::string pv(VCI_PV_CHARS, 'A');
    // k_vcc_records
    std::map<std::string, uint32_t> rank_of;          // the directory's DIDs and their ranks in byte order
    for (uint32_t d = 0; d < dir_n; d++) rank_of[std::string((const char*)dir_dids + dir_off[d], dir_off[d + 1] - dir_off[d])] = 0;
    { uint32_t r = 0; for (auto& e : rank_of) e.second = r++; }
    std::vector<uint32_t> by_rank(dir_n);
    for (uint32_t d = 0; d < dir_n; d++) by_rank[rank_of[std::string((const char*)dir_dids + dir_off[d], dir_off[d + 1] - dir_off[d])]] = d;
    std::set<uint32_t> distinct;
    bool host = false;
    auto take = [&](VccStr s) {
        if (!vcc_did_wanted(s.p, s.len)) return;
        auto f = rank_of.find(std::string((const char*)s.p, s.len));
        if (f == rank_of.end()) return;
        distinct.insert(f->second);
        host |= s.len > VCC_DID_MAX;
    };
    std::vector<VccRecord> recs(cnt);
    std::vector<uint64_t> rlen(cnt + 1, 0);
    for (uint32_t k = 0; k < cnt; k++) {
        VccRecord& x = recs[k];
        x.vc_id.p = rec_cols + rec_coff[2 * k]; x.vc_id.len = rec_coff[2 * k + 1] - rec_coff[2 * k];
        x.status.p = rec_cols + rec_coff[2 * k + 1]; x.status.len = rec_coff[2 * k + 2] - rec_coff[2 * k + 1];
        x.cols = crec_cols; x.coff = crec_coff + VCC_REC_COLUMNS * k;
        x.flags = flags[k]; x.doc_size = doc_size[k]; x.sec = created[2 * k]; x.nsec = created[2 * k + 1]; x.zone = zone[k];
        if (vcc_record_state(x) == VCC_HOST) { host = true; continue; }
        ByteCounter c; c.init();
        vcc_record(c, x);
        rlen[k + 1] = rlen[k] + c.n + (k ? 1 : 0);
        take(x.col(VCC_R_ISSUER)); take(x.col(VCC_R_CALLER)); take(x.col(VCC_R_TARGET));
    }
    VccStr issuer; issuer.p = cols + coff[VCW_COL_ISSUER]; issuer.len = coff[VCW_COL_ISSUER + 1] - coff[VCW_COL_ISSUER];
    take(issuer);
    VccStr resolved; resolved.p = chain_cols + chain_coff[VCC_COL_RESOLVED_AT]; resolved.len = chain_coff[VCC_COL_RESOLVED_AT + 1] - chain_coff[VCC_COL_RESOLVED_AT];
    // k_vcc_sizes
    VccFrame f;
    auto col = [&](uint32_t c) { VccStr s; s.p = cols + coff[c]; s.len = coff[c + 1] - coff[c]; return s; };
    f.workflow_id = col(VCW_COL_WORKFLOW); f.session_id = col(VCW_COL_SESSION); f.issuer = issuer;
    f.wf_vc_id.p = chain_cols + chain_coff[0]; f.wf_vc_id.len = chain_coff[1] - chain_coff[0];
    f.status = p.status; f.cnt = cnt; f.completed = p.completed;
    for (int t = 0; t < 3; t++) f.snap[t] = clock[t];
    if (cnt) { f.start[0] = created[2 * p.start]; f.start[1] = created[2 * p.start + 1]; f.start[2] = zone[p.start]; }
    else for (int t = 0; t < 3; t++) f.start[t] = clock[t];
    f.has_end = p.end != VCW_NONE;
    f.end[0] = f.has_end ? created[2 * p.end] : 0; f.end[1] = f.has_end ? created[2 * p.end + 1] : 0; f.end[2] = f.has_end ? zone[p.end] : 0;
    f.has_bundle = !distinct.empty();
    f.proof_value = (const uint8_t*)pv.data();
    f.doc_len = doc_len;
    if (host || !vcc_time_ok(clock[0], clock[1], clock[2]) || resolved.len > VCC_RESOLVED_MAX) { *state = VCC_HOST; return 0; }
    *state = VCC_BUILT;
    const uint32_t zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    std::vector<uint64_t> elen(distinct.size() + 1, 0);
    std::vector<uint32_t> ents(distinct.begin(), distinct.end());
    for (size_t k = 0; k < ents.size(); k++) {
        const uint32_t d = by_rank[ents[k]];
        VccStr did; did.p = dir_dids + dir_off[d]; did.len = dir_off[d + 1] - dir_off[d];
        ByteCounter c; c.init();
        vcc_entry(c, did, zero, resolved);
        elen[k + 1] = elen[k] + c.n + (k ? 1 : 0);
    }
    uint64_t L[VCC_PARTS], at[VCC_PARTS];
    for (uint32_t q = 0; q < VCC_PARTS; q++) { ByteCounter c; c.init(); vcc_frame(c, f, q); L[q] = c.n; }
    at[0] = 0;
    const uint64_t rec_at = L[0];
    at[1] = rec_at + rlen[cnt];
    const uint64_t ids_at = at[1] + L[1] - 1;
    at[2] = ids_at + p.ids_bytes - 1;
    const uint64_t doc_at = at[2] + L[2];
    at[3] = doc_at + doc_len;
    const uint64_t ent_at = at[3] + L[3];
    at[4] = ent_at + elen[ents.size()];
    *body_len = at[4] + L[4];
    if (!body) return 0;
    // the emit passes
    for (uint32_t q = 0; q < VCC_PARTS; q++) { ByteWriter w; w.init(body + at[q]); vcc_frame(w, f, q); w.finish(); }
    uint64_t before = 0;
    for (uint32_t k = 0; k < cnt; k++) {
        {
            ByteWriter w; w.init(body + rec_at + rlen[k]);
            if (k) w.put(',');
            vcc_record(w, recs[k]);
            w.finish();
        }
        ByteWriter w; w.init(body + ids_at + vcw_id_at(before, k));
        if (k) w.put(',');
        w.put('"');
        go_json_escape(w, recs[k].vc_id.p, recs[k].vc_id.len);
        w.put('"');
        w.finish();
        before += id_len[k];
    }
    for (size_t k = 0; k < ents.size(); k++) {
        const uint32_t d = by_rank[ents[k]];
        VccStr did; did.p = dir_dids + dir_off[d]; did.len = dir_off[d + 1] - dir_off[d];
        uint32_t pk[8];
        memcpy(pk, dir_pks + 32 * (size_t)d, 32);
        ByteWriter w; w.init(body + ent_at + elen[k]);
        if (k) w.put(',');
        vcc_entry(w, did, pk, resolved);
        w.finish();
    }
    memcpy(body + doc_at, doc.data(), doc_len);
    return 0;
}

uint32_t hs_vcc_did_wanted(const uint8_t* d, uint64_t len) { return vcc_did_wanted(d, len); }

// time.Time.MarshalJSON of (seconds, nanoseconds, zone); returns the length (0 when vcc_time_ok declines)
uint32_t hs_vcc_time(int64_t sec, int64_t nsec, int64_t zone, uint8_t* out) {
    if (!vcc_time_ok(sec, nsec, zone)) return 0;
    ByteCounter c; c.init();
    vcc_put_time(c, sec, nsec, zone);
    ByteWriter w; w.init(out);
    vcc_put_time(w, sec, nsec, zone);
    w.finish();
    return (uint32_t)c.n;
}

}  // extern "C"
