// TEST-ONLY CPU build of the DID resolution routines (agentfield_b200/csrc/afc_didresolve.cuh): what a thread of k_dres_entries and
// k_dres_canon does for one directory entry, and what a thread of k_dres_probe and k_dres_emit does for one request.  The directory probe
// is the caller's (a Python dict).  Compiled on its own by tests/test_didresolve_hostsim.py.
#define AFC_HOSTSIM 1
#include <vector>

#include "../../agentfield_b200/csrc/afc_didresolve.cuh"

using namespace afc;

static DresStr S(const uint8_t* p, uint64_t n) { DresStr s; s.p = p; s.len = n; return s; }

extern "C" {

// One entry: out = {resolve length, document length, side length}; when side is given (out[2] + 32 bytes) and out[2] > 0, the
// canonical JWK text k_dres_canon writes there.
void hs_dres_entry(uint32_t kind, const uint8_t* did, uint64_t dl, const uint8_t* path, uint64_t pl, const uint8_t* fn, uint64_t fl,
                   const uint8_t* jwk, uint64_t jl, uint32_t* out, uint8_t* side) {
    std::vector<uint32_t> tape(jl / 2 + 1);
    const DresEntry e = dres_entry(kind, S(did, dl), S(path, pl), S(fn, fl), S(jwk, jl), tape.data());
    out[0] = e.rlen; out[1] = e.dlen; out[2] = e.side;
    if (side && e.side) {
        ByteWriter w; w.init(side);
        jv_emit(w, jwk, (uint32_t)jl, tape.data());
        w.finish();
    }
}

// One request (req_kind, req) answered by the entry (found) with its cached lengths and its side text (sl == 0: the stored JWK):
// *state and *len as k_dres_probe writes them and, when body is given (*len plus 32 bytes), the body k_dres_emit writes.
void hs_dres_request(uint32_t req_kind, const uint8_t* req, uint64_t rl, int found, uint32_t kind, const uint8_t* did, uint64_t dl,
                     const uint8_t* path, uint64_t pl, const uint8_t* fn, uint64_t fl, const uint8_t* jwk, uint64_t jl, const uint8_t* side,
                     uint64_t sl, uint32_t rlen, uint32_t dlen, uint32_t* state, uint8_t* body, uint64_t* len) {
    uint32_t st;
    uint64_t n;
    if (req_kind > DRES_DOCUMENT) { st = DRES_HOST; n = 0; }
    else if (rl == 0) { st = DRES_BAD_REQUEST; n = DRES_BAD_REQUEST_LEN; }
    else if (!found) {
        ByteCounter c; c.init();
        dres_not_found(c, req_kind, S(req, rl));
        st = DRES_NOT_FOUND; n = c.n;
    } else {
        n = req_kind == DRES_RESOLVE ? rlen : dlen;
        st = n ? DRES_FOUND : DRES_HOST;
    }
    *state = st; *len = n;
    if (!body || st == DRES_HOST) return;
    ByteWriter w; w.init(body);
    if (st == DRES_BAD_REQUEST) vci_put_text(w, DRES_BAD_REQUEST_BODY);
    else if (st == DRES_NOT_FOUND) dres_not_found(w, req_kind, S(req, rl));
    else if (req_kind == DRES_RESOLVE) dres_resolve(w, kind, S(did, dl), S(path, pl), S(fn, fl), S(jwk, jl));
    else dres_document(w, S(did, dl), sl ? S(side, sl) : S(jwk, jl));
    w.finish();
}

uint64_t hs_dres_request_fixed() { return DRES_DOC404_FIXED; }

}
