// TEST-ONLY CPU build of the webhook routines (agentfield_b200/csrc/afc_float.cuh, afc_jsonval.cuh, afc_webhook.cuh): what one thread of
// k_wh_sizes, k_wh_emit and k_wh_sign does.  Compiled on its own by tests/test_webhook_hostsim.py.
#define AFC_HOSTSIM 1
#include "../../agentfield_b200/csrc/afc_webhook.cuh"

#include <vector>

using namespace afc;

extern "C" {

// strconv.ParseFloat of a JSON number token: 1 and the bits, or 0 (declined)
int hs_fl_parse(const uint8_t* s, uint32_t len, uint64_t* bits) { return fl_parse(s, len, bits) ? 1 : 0; }

// encoding/json's text of a float64 (finite, zero or normal); returns its length (out: at least 32 bytes)
uint32_t hs_fl_format(uint64_t bits, uint8_t* out) {
    ByteCounter c; c.init();
    fl_put(c, bits);
    ByteWriter w; w.init(out);
    fl_put(w, bits);
    w.finish();
    return (uint32_t)c.n;
}

// many tokens (packed, n + 1 offsets): ok[i] and bits[i]
void hs_fl_parse_batch(const uint8_t* s, const uint64_t* off, uint32_t n, uint8_t* ok, uint64_t* bits) {
    for (uint32_t i = 0; i < n; i++) ok[i] = fl_parse(s + off[i], (uint32_t)(off[i + 1] - off[i]), bits + i) ? 1 : 0;
}
// many values: 32 bytes of text per value at out + 32 i, lengths in len
void hs_fl_format_batch(const uint64_t* bits, uint32_t n, uint8_t* out, uint8_t* len) {
    for (uint32_t i = 0; i < n; i++) {
        uint8_t tmp[64];
        len[i] = (uint8_t)hs_fl_format(bits[i], tmp);
        memcpy(out + 32ull * i, tmp, 32);
    }
}

uint32_t hs_jv_validate(const uint8_t* d, uint64_t len) { return jv_validate(d, len); }

// json.Marshal(json.Unmarshal(d)) of a valid text: its length, or -1 (declined), -2 (the two passes disagree), -3 (out too small)
int64_t hs_jv_emit(const uint8_t* d, uint32_t len, uint8_t* out, uint64_t cap) {
    std::vector<uint32_t> tape(len / 2 + 1);
    ByteCounter c; c.init();
    if (!jv_emit(c, d, len, tape.data())) return -1;
    if (c.n + 32 > cap) return -3;
    ByteWriter w; w.init(out);
    if (!jv_emit(w, d, len, tape.data())) return -2;
    w.finish();
    ByteCounter c2; c2.init();
    jv_emit(c2, d, len, tape.data());
    return c2.n == c.n ? (int64_t)c.n : -2;
}

// One delivery: returns the body length (and writes the body and, with a secret, the header), or -1 for WH_HOST, -3 for a too small out
int64_t hs_wh_delivery(const uint8_t* cols, const uint64_t* coff, int64_t duration, uint32_t flags, const uint8_t* result, uint64_t result_len,
                       const uint8_t* key, uint32_t klen, uint8_t* out, uint64_t cap, uint8_t* header) {
    WhItem it{cols, coff, duration, flags, result, result_len};
    const uint32_t plan = wh_plan(it);
    if (plan & WH_P_HOST) return -1;
    std::vector<uint32_t> tape(result_len / 2 + 1);
    ByteCounter c; c.init();
    if (!wh_body(c, it, plan, tape.data())) return -1;
    if (c.n + 32 > cap) return -3;
    ByteWriter w; w.init(out);
    wh_body(w, it, plan, tape.data());
    w.finish();
    if (flags & WH_HAS_SECRET) {
        uint32_t st[8];
        uint8_t mac[32];
        hmac_sha256_msg(st, key, klen, out, c.n);
        store_digest256(mac, st);
        wh_header_text(header, mac);
    }
    return (int64_t)c.n;
}

uint64_t hs_wh_fixed_bytes() { return wh_fixed_bytes(); }

}  // extern "C"
