/* tests/c_abi/vc_chain.c — a plain-C caller of afc_did_directory_new and afc_vc_workflow_chain_batch (include/afcrypto.h), compiled as
 * C99 with -pedantic against the header alone, as cgo would.  Checks: the bound is additive over workflows and covers the bodies; the
 * AFC_EINVAL cases (NULL pointers, a bodies_cap one byte short, a duplicate DID in the directory, directory offsets and record offsets
 * that run backwards, more DID occurrence slots than the kernels count, a directory of another context); n = 0; and that two workflows
 * (one without records, one with two records whose DIDs the directory holds) come back built, with the bundle's members in byte order.
 * Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_vcchain_c_abi.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "afcrypto.h"

#define N 2
#define M 2

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
    uint8_t seeds[32], exp[96];
    for (int i = 0; i < 32; i++) seeds[i] = (uint8_t)(i * 7 + 1);
    if (afc_ed25519_expand_batch(ctx, seeds, 1, exp) != AFC_OK) { fprintf(stderr, "expand\n"); return 3; }

    /* the directory: three DIDs, keys of any 32 bytes */
    static uint8_t dids[256], pks[3 * 32];
    uint64_t did_off[4] = {0};
    put(dids, did_off, 0, "did:key:zIssuer");
    put(dids, did_off, 1, "did:web:example.com");
    put(dids, did_off, 2, "did:key:zCaller");
    for (int i = 0; i < 96; i++) pks[i] = (uint8_t)i;
    afc_did_directory* dir = NULL;
    CHECK(afc_did_directory_new(NULL, pks, dids, did_off, 3, &dir) == AFC_EINVAL);
    CHECK(afc_did_directory_new(ctx, NULL, dids, did_off, 3, &dir) == AFC_EINVAL);
    CHECK(afc_did_directory_new(ctx, pks, NULL, did_off, 3, &dir) == AFC_EINVAL);
    CHECK(afc_did_directory_new(ctx, pks, dids, NULL, 3, &dir) == AFC_EINVAL);
    {
        uint64_t dup[3] = {0, 15, 30};
        static uint8_t two[32];
        memcpy(two, "did:key:zIssuerdid:key:zIssuer", 30);
        CHECK(afc_did_directory_new(ctx, pks, two, dup, 2, &dir) == AFC_EINVAL);
        uint64_t back[4] = {0, 15, 10, 20};
        CHECK(afc_did_directory_new(ctx, pks, dids, back, 3, &dir) == AFC_EINVAL);
    }
    CHECK(afc_did_directory_new(ctx, pks, dids, did_off, 3, &dir) == AFC_OK && dir);

    /* two workflows: none, and two records */
    static uint8_t cols[1024], rcols[256], ccols[256], crcols[2048];
    uint64_t col_off[N * AFC_WORKFLOW_COLUMNS + 1] = {0}, rec_off[N + 1] = {0, 0, M}, rec_col_off[2 * M + 1] = {0};
    uint64_t ccol_off[N * AFC_CHAIN_WORKFLOW_COLUMNS + 1] = {0}, crcol_off[M * AFC_CHAIN_RECORD_COLUMNS + 1] = {0};
    const char* wcols[AFC_WORKFLOW_COLUMNS] = {"wf", "sess", "did:key:zIssuer", "vc-wf", "2026-09-21T06:00:00Z", "2026-09-21T06:00:05Z",
                                               "2026-09-21T06:00:06Z"};
    size_t k = 0;
    for (int i = 0; i < N; i++)
        for (int c = 0; c < AFC_WORKFLOW_COLUMNS; c++, k++) put(cols, col_off, k, wcols[c]);
    put(rcols, rec_col_off, 0, "vc-1"); put(rcols, rec_col_off, 1, "succeeded");
    put(rcols, rec_col_off, 2, "vc-2"); put(rcols, rec_col_off, 3, "failed");
    for (k = 0; k < (size_t)N * AFC_CHAIN_WORKFLOW_COLUMNS; k++) put(ccols, ccol_off, k, k % 2 ? "2026-09-21T06:00:07Z" : "vc-chain");
    const char* rc13[AFC_CHAIN_RECORD_COLUMNS] = {"exec", "wf", "sess", "agent", "name", "did:key:zIssuer", "did:web:example.com", "did:key:zCaller",
                                                  "{ \"a\" : 1 }", "sig", "", "in", "out"};
    for (k = 0; k < (size_t)M * AFC_CHAIN_RECORD_COLUMNS; k++) put(crcols, crcol_off, k, rc13[k % AFC_CHAIN_RECORD_COLUMNS]);
    int64_t created[2 * M] = {1790000000, 0, 1790000001, 500000000}, clock[3 * N] = {1790000100, 0, 0, 1790000100, 7, 3600};
    int64_t size[M] = {11, 11};
    int32_t zone[M] = {0, -28800};
    uint8_t flags[M] = {0, AFC_CHAIN_WORKFLOW_NAME_NIL};
    uint32_t ki[N] = {0, 0};

    const uint64_t b0 = afc_vc_workflow_chain_bound(col_off, rec_off, rec_col_off, ccol_off, crcol_off, 1);
    const uint64_t b1 = afc_vc_workflow_chain_bound(col_off + AFC_WORKFLOW_COLUMNS, rec_off + 1, rec_col_off, ccol_off + AFC_CHAIN_WORKFLOW_COLUMNS,
                                                    crcol_off, 1);
    const uint64_t cap = afc_vc_workflow_chain_bound(col_off, rec_off, rec_col_off, ccol_off, crcol_off, N);
    CHECK(cap == b0 + b1 && b0 > 0 && b1 > b0);
    CHECK(afc_vc_workflow_chain_bound(NULL, rec_off, rec_col_off, ccol_off, crcol_off, N) == 0);
    CHECK(afc_vc_workflow_chain_bound(col_off, rec_off, rec_col_off, ccol_off, crcol_off, 0) == 0);
    uint8_t* bodies = (uint8_t*)malloc(cap);
    uint64_t body_off[N + 1];
    uint8_t state[N];
#define CALL(ctx_, exp_, cols_, rec_off_, dir_, n_, bodies_, cap_, body_off_, state_) \
    afc_vc_workflow_chain_batch(ctx_, exp_, 1, ki, cols_, col_off, rec_off_, rcols, rec_col_off, created, ccols, ccol_off, clock, crcols, \
                                crcol_off, flags, size, zone, dir_, n_, bodies_, cap_, body_off_, state_)
    CHECK(CALL(NULL, exp, cols, rec_off, dir, N, bodies, cap, body_off, state) == AFC_EINVAL);
    CHECK(CALL(ctx, NULL, cols, rec_off, dir, N, bodies, cap, body_off, state) == AFC_EINVAL);
    CHECK(CALL(ctx, exp, NULL, rec_off, dir, N, bodies, cap, body_off, state) == AFC_EINVAL);
    CHECK(CALL(ctx, exp, cols, rec_off, NULL, N, bodies, cap, body_off, state) == AFC_EINVAL);
    CHECK(CALL(ctx, exp, cols, rec_off, dir, N, NULL, cap, body_off, state) == AFC_EINVAL);
    CHECK(CALL(ctx, exp, cols, rec_off, dir, N, bodies, cap, body_off, NULL) == AFC_EINVAL);
    CHECK(CALL(ctx, exp, cols, rec_off, dir, N, bodies, cap - 1, body_off, state) == AFC_EINVAL);
    {
        uint64_t back[N + 1] = {0, M, 0};
        CHECK(CALL(ctx, exp, cols, back, dir, N, bodies, cap, body_off, state) == AFC_EINVAL);
        uint64_t huge[N + 1] = {0, 0, 0x2aaaaaabull};              /* 3 x records + workflows past 2^31 - 1: refused before any read */
        CHECK(CALL(ctx, exp, cols, huge, dir, N, bodies, cap, body_off, state) == AFC_EINVAL);
    }
    if (afc_init(0, &ctx2) == AFC_OK) {
        afc_did_directory* other = NULL;
        CHECK(afc_did_directory_new(ctx2, pks, dids, did_off, 3, &other) == AFC_OK);
        CHECK(CALL(ctx, exp, cols, rec_off, other, N, bodies, cap, body_off, state) == AFC_EINVAL);
        afc_did_directory_free(other);
        afc_destroy(ctx2);
    }
    body_off[0] = 99;
    CHECK(CALL(ctx, exp, cols, rec_off, dir, 0, bodies, 0, body_off, state) == AFC_OK && body_off[0] == 0);

    CHECK(CALL(ctx, exp, cols, rec_off, dir, N, bodies, cap, body_off, state) == AFC_OK);
    CHECK(state[0] == AFC_CHAIN_BUILT && state[1] == AFC_CHAIN_BUILT);
    CHECK(body_off[0] == 0 && body_off[2] <= cap);
    if (!bad) {
        const char* b = (const char*)bodies;
        CHECK(memcmp(b, "{\"workflow_id\":\"wf\",\"component_vcs\":[],", 39) == 0);
        const char* second = b + body_off[1];
        char* text = (char*)calloc(body_off[2] - body_off[1] + 1, 1);
        memcpy(text, second, body_off[2] - body_off[1]);
        const char* a = strstr(text, "\"did:key:zCaller\":{\"method\":\"key\"");
        const char* c = strstr(text, "\"did:key:zIssuer\":{\"method\":\"key\"");
        const char* w = strstr(text, "\"did:web:example.com\":{\"method\":\"web\"");
        CHECK(a && c && w && a < c && c < w);
        CHECK(strstr(text, "\"vc_document\":{\"a\":1}") != NULL);
        CHECK(strstr(text, "\"created_at\":\"2026-09-21T06:13:21.5-08:00\"") != NULL);
        CHECK(strstr(text, "\"snapshot_time\":\"2026-09-21T15:15:00.000000007+01:00\"") != NULL);
        free(text);
    }
    free(bodies);
    afc_did_directory_free(dir);
    afc_destroy(ctx);
    if (bad) return 1;
    printf("vc_chain ok\n");
    return 0;
}
