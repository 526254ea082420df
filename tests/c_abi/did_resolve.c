/* tests/c_abi/did_resolve.c — a plain-C caller of afc_did_directory_set_identities and afc_did_resolve_batch[_dev] (include/afcrypto.h),
 * compiled as C99 with -pedantic against the header alone, as cgo would.  Checks: the bound is additive over requests and covers the
 * bodies; the AFC_EINVAL cases (NULL pointers, a second set_identities, a kind out of range, identity offsets that run backwards, a
 * directory without identities, a directory of another context, a bodies_cap one byte short, request offsets that run backwards, a
 * request of 2^31 bytes); n = 0; and the states of four requests (found, not found, empty, a document whose stored JWK is an array).
 * Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_didresolve_c_abi.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "afcrypto.h"

static void put(uint8_t* buf, uint64_t* off, size_t k, const char* s) {
    memcpy(buf + off[k], s, strlen(s));
    off[k + 1] = off[k] + strlen(s);
}

int main(void) {
    afc_ctx *ctx = NULL, *ctx2 = NULL;
    int rc = afc_init(0, &ctx);
    if (rc == AFC_ECUDA) { printf("no usable GPU: %s (the library has no CPU path)\n", afc_strerror(rc)); return 77; }
    if (rc != AFC_OK) { fprintf(stderr, "afc_init: %s\n", afc_strerror(rc)); return 2; }
    int bad = 0;
#define CHECK(c) do { if (!(c)) { fprintf(stderr, "line %d: %s\n", __LINE__, #c); bad = 1; } } while (0)

    static uint8_t dids[256], pks[2 * 32], cols[512];
    uint64_t did_off[3] = {0}, col_off[7] = {0};
    put(dids, did_off, 0, "did:key:zRoot");
    put(dids, did_off, 1, "did:key:zAgent");
    uint8_t kinds[2] = {AFC_DID_KIND_SERVER, AFC_DID_KIND_AGENT};
    put(cols, col_off, 0, "m/44'/0'");
    put(cols, col_off, 1, "");
    put(cols, col_off, 2, "{\"alg\":\"EdDSA\",\"x\":\"abc\"}");
    put(cols, col_off, 3, "m/44'/1'/0'");
    put(cols, col_off, 4, "");
    put(cols, col_off, 5, "[1]");
    afc_did_directory *dir = NULL, *plain = NULL;
    CHECK(afc_did_directory_new(ctx, pks, dids, did_off, 2, &dir) == AFC_OK && dir);
    CHECK(afc_did_directory_new(ctx, pks, dids, did_off, 2, &plain) == AFC_OK && plain);
    CHECK(afc_did_directory_set_identities(NULL, kinds, cols, col_off) == AFC_EINVAL);
    CHECK(afc_did_directory_set_identities(dir, NULL, cols, col_off) == AFC_EINVAL);
    CHECK(afc_did_directory_set_identities(dir, kinds, cols, NULL) == AFC_EINVAL);
    {
        uint8_t k5[2] = {0, 4};
        CHECK(afc_did_directory_set_identities(dir, k5, cols, col_off) == AFC_EINVAL);
        uint64_t back[7] = {0, 8, 4, 30, 40, 40, 43};
        CHECK(afc_did_directory_set_identities(dir, kinds, cols, back) == AFC_EINVAL);
    }
    CHECK(afc_did_directory_set_identities(dir, kinds, cols, col_off) == AFC_OK);
    CHECK(afc_did_directory_set_identities(dir, kinds, cols, col_off) == AFC_EINVAL);     /* once per directory */

    /* four requests: resolve the root, document an unknown DID, resolve "", document the agent (its JWK is an array: HOST) */
    static uint8_t reqs[256];
    uint64_t req_off[5] = {0};
    put(reqs, req_off, 0, "did:key:zRoot");
    put(reqs, req_off, 1, "did:key:zNone<");
    put(reqs, req_off, 2, "");
    put(reqs, req_off, 3, "did:key:zAgent");
    uint8_t rk[4] = {AFC_DIDRES_RESOLVE, AFC_DIDRES_DOCUMENT, AFC_DIDRES_RESOLVE, AFC_DIDRES_DOCUMENT};
    const uint64_t cap = afc_did_resolve_bound(dir, req_off, 4);
    CHECK(cap > 0 && afc_did_resolve_bound(plain, req_off, 4) == 0 && afc_did_resolve_bound(dir, req_off, 0) == 0);
    CHECK(cap == afc_did_resolve_bound(dir, req_off, 2) + afc_did_resolve_bound(dir, req_off + 2, 2));      /* additive */
    CHECK(cap == afc_did_resolve_bound(dir, req_off, 1) + afc_did_resolve_bound(dir, req_off + 1, 3));
    uint8_t* bodies = (uint8_t*)malloc(cap);
    uint64_t body_off[5] = {0};
    uint8_t state[4] = {9, 9, 9, 9};
    CHECK(afc_did_resolve_batch(NULL, dir, rk, reqs, req_off, 4, bodies, cap, body_off, state) == AFC_EINVAL);
    CHECK(afc_did_resolve_batch(ctx, NULL, rk, reqs, req_off, 4, bodies, cap, body_off, state) == AFC_EINVAL);
    CHECK(afc_did_resolve_batch(ctx, dir, NULL, reqs, req_off, 4, bodies, cap, body_off, state) == AFC_EINVAL);
    CHECK(afc_did_resolve_batch(ctx, dir, rk, NULL, req_off, 4, bodies, cap, body_off, state) == AFC_EINVAL);
    CHECK(afc_did_resolve_batch(ctx, dir, rk, reqs, NULL, 4, bodies, cap, body_off, state) == AFC_EINVAL);
    CHECK(afc_did_resolve_batch(ctx, dir, rk, reqs, req_off, 4, NULL, cap, body_off, state) == AFC_EINVAL);
    CHECK(afc_did_resolve_batch(ctx, dir, rk, reqs, req_off, 4, bodies, cap, NULL, state) == AFC_EINVAL);
    CHECK(afc_did_resolve_batch(ctx, dir, rk, reqs, req_off, 4, bodies, cap, body_off, NULL) == AFC_EINVAL);
    CHECK(afc_did_resolve_batch(ctx, plain, rk, reqs, req_off, 4, bodies, cap, body_off, state) == AFC_EINVAL);   /* no identities */
    CHECK(afc_did_resolve_batch(ctx, dir, rk, reqs, req_off, 4, bodies, cap - 1, body_off, state) == AFC_EINVAL);
    {
        uint64_t back[5] = {0, 13, 10, 27, 27};
        CHECK(afc_did_resolve_batch(ctx, dir, rk, reqs, back, 4, bodies, cap + 100, body_off, state) == AFC_EINVAL);
        uint64_t huge[2] = {0, 1ull << 31};                      /* checked before any byte is read */
        CHECK(afc_did_resolve_batch(ctx, dir, rk, reqs, huge, 1, bodies, afc_did_resolve_bound(dir, huge, 1), body_off, state) == AFC_EINVAL);
    }
    if (afc_init(0, &ctx2) == AFC_OK) {
        CHECK(afc_did_resolve_batch(ctx2, dir, rk, reqs, req_off, 4, bodies, cap, body_off, state) == AFC_EINVAL);
        afc_destroy(ctx2);
    }
    {
        uint64_t z = 77;
        CHECK(afc_did_resolve_batch(ctx, dir, NULL, NULL, req_off, 0, NULL, 0, &z, NULL) == AFC_OK && z == 0);
    }
    CHECK(afc_did_resolve_batch(ctx, dir, rk, reqs, req_off, 4, bodies, cap, body_off, state) == AFC_OK);
    CHECK(state[0] == AFC_DIDRES_FOUND && state[1] == AFC_DIDRES_NOT_FOUND && state[2] == AFC_DIDRES_BAD_REQUEST && state[3] == AFC_DIDRES_HOST);
    CHECK(body_off[4] <= cap && body_off[4] == body_off[3]);
    {
        const char* want1 = "{\"details\":\"DID not found: did:key:zNone\\u003c\",\"error\":\"DID not found\"}";
        const char* want2 = "{\"error\":\"DID parameter is required\"}";
        CHECK(body_off[2] - body_off[1] == strlen(want1) && memcmp(bodies + body_off[1], want1, strlen(want1)) == 0);
        CHECK(body_off[3] - body_off[2] == strlen(want2) && memcmp(bodies + body_off[2], want2, strlen(want2)) == 0);
        const char* want0 = "{\"component_type\":\"agentfield_server\",\"derivation_path\":\"m/44'/0'\",\"did\":\"did:key:zRoot\",\"function_name\":\"\","
                            "\"public_key_jwk\":\"{\\\"alg\\\":\\\"EdDSA\\\",\\\"x\\\":\\\"abc\\\"}\"}";
        CHECK(body_off[1] == strlen(want0) && memcmp(bodies, want0, strlen(want0)) == 0);
    }
    {
        /* the _dev call's argument checks and n = 0 return before any device access (the header declares no device allocator; the GPU
           tests run the _dev call on device buffers) */
        CHECK(afc_did_resolve_batch_dev(ctx, plain, rk, reqs, req_off, 4, bodies, cap, body_off, state, NULL) == AFC_EINVAL);
        CHECK(afc_did_resolve_batch_dev(ctx, dir, rk, reqs, req_off, 0, bodies, cap, body_off, state, NULL) == AFC_OK);
    }
    free(bodies);
    afc_did_directory_free(dir);
    afc_did_directory_free(plain);
    afc_destroy(ctx);
    if (bad) return 1;
    printf("did_resolve ok\n");
    return 0;
}
