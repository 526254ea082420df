/* tests/c_abi/workflow_vc.c — a plain-C caller of afc_vc_issue_workflow_batch (include/afcrypto.h), compiled as C99 with -pedantic
 * against the header alone, as cgo would: two issuers, four workflows (no records; two succeeded records; a failed and a running record
 * with an id that needs escaping; a status that is not ASCII, which the caller must build itself), issued in one call.  Every built
 * document must verify through afc_vc_verify_stored_batch(AFC_DOC_WORKFLOW_VC), end in its proofValue, and its summary must match.
 * Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_vcworkflow_c_abi.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "afcrypto.h"

static size_t b64url(const uint8_t* in, size_t n, char* out) {
    const char* a = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789-_";
    size_t o = 0, i;
    for (i = 0; i + 3 <= n; i += 3) {
        uint32_t v = (uint32_t)in[i] << 16 | (uint32_t)in[i + 1] << 8 | in[i + 2];
        out[o++] = a[v >> 18]; out[o++] = a[(v >> 12) & 63]; out[o++] = a[(v >> 6) & 63]; out[o++] = a[v & 63];
    }
    if (n - i == 1) {
        uint32_t v = (uint32_t)in[i] << 16;
        out[o++] = a[v >> 18]; out[o++] = a[(v >> 12) & 63];
    } else if (n - i == 2) {
        uint32_t v = (uint32_t)in[i] << 16 | (uint32_t)in[i + 1] << 8;
        out[o++] = a[v >> 18]; out[o++] = a[(v >> 12) & 63]; out[o++] = a[(v >> 6) & 63];
    }
    return o;
}

#define N 4
#define K 2
#define R 5

int main(void) {
    afc_ctx* ctx = NULL;
    int rc = afc_init(0, &ctx);
    if (rc == AFC_ECUDA) { printf("no usable GPU: %s (the library has no CPU path)\n", afc_strerror(rc)); return 77; }
    if (rc != AFC_OK) { fprintf(stderr, "afc_init: %s\n", afc_strerror(rc)); return 2; }
    int bad = 0;
    uint8_t seeds[K * 32], exp[K * 96], pks[K * 32];
    for (int i = 0; i < K * 32; i++) seeds[i] = (uint8_t)(i * 11 + 5);
    if (afc_ed25519_expand_batch(ctx, seeds, K, exp) != AFC_OK) { fprintf(stderr, "expand\n"); return 3; }
    char dids[K][64];
    uint8_t didbuf[K * 64];
    uint64_t did_off[K + 1] = {0};
    for (int k = 0; k < K; k++) {
        uint8_t raw[34] = {0xed, 0x01};
        memcpy(pks + 32 * k, exp + 96 * k + 64, 32);
        memcpy(raw + 2, pks + 32 * k, 32);
        strcpy(dids[k], "did:key:z");
        dids[k][9 + b64url(raw, 34, dids[k] + 9)] = 0;
        memcpy(didbuf + did_off[k], dids[k], strlen(dids[k]));
        did_off[k + 1] = did_off[k] + strlen(dids[k]);
    }
    /* the columns, AFC_WORKFLOW_COLUMNS per workflow */
    static uint8_t cols[4096];
    uint64_t col_off[N * AFC_WORKFLOW_COLUMNS + 1] = {0};
    uint32_t ki[N];
    for (int i = 0; i < N; i++) {
        char wf[16];
        sprintf(wf, "wf_%d", i);
        const char* c[AFC_WORKFLOW_COLUMNS] = {wf, i ? "sess_1" : "", dids[i % K], "vc-1790000000000000001", "2026-09-21T06:00:00Z",
                                               "2026-09-21T06:00:05Z", "2026-09-21T06:00:06Z"};
        ki[i] = (uint32_t)(i % K);
        for (int k = 0; k < AFC_WORKFLOW_COLUMNS; k++) {
            const size_t j = (size_t)i * AFC_WORKFLOW_COLUMNS + k;
            memcpy(cols + col_off[j], c[k], strlen(c[k]));
            col_off[j + 1] = col_off[j] + strlen(c[k]);
        }
    }
    /* records: workflow 0 none, 1: two succeeded, 2: failed + running (escaped id), 3: a non-ASCII status */
    uint64_t rec_off[N + 1] = {0, 0, 2, 4, 5};
    const char* rec[R][2] = {{"vc-11", "succeeded"}, {"vc-12", " Done "}, {"vc-21", "failed"}, {"vc-\"22\"<&>", "in_progress"},
                             {"vc-31", "d\xc3\xb6ne"}};
    int64_t created[2 * R] = {1790000000, 5, 1790000000, 4, 1790000100, 0, 1790000050, 999999999, 1790000000, 0};
    static uint8_t rec_cols[512];
    uint64_t rec_col_off[2 * R + 1] = {0};
    for (int j = 0; j < 2 * R; j++) {
        const char* s = rec[j / 2][j % 2];
        memcpy(rec_cols + rec_col_off[j], s, strlen(s));
        rec_col_off[j + 1] = rec_col_off[j] + strlen(s);
    }
    const uint64_t cap = afc_vc_workflow_bound(col_off, rec_off, rec_col_off, N);
    uint8_t* docs = (uint8_t*)malloc(cap);
    uint64_t doc_off[N + 1];
    uint8_t pv[N * 86], state[N];
    uint32_t summary[N * 4];
    rc = afc_vc_issue_workflow_batch(ctx, exp, K, ki, cols, col_off, rec_off, rec_cols, rec_col_off, created, N, docs, cap, doc_off, pv, state,
                                     summary);
    if (rc != AFC_OK) { fprintf(stderr, "issue: %s\n", afc_strerror(rc)); return 4; }
    if (afc_vc_issue_workflow_batch(ctx, exp, K, ki, cols, col_off, rec_off, rec_cols, rec_col_off, created, N, docs, cap - 1, doc_off, pv, state,
                                    summary) != AFC_EINVAL) { printf("bound not enforced\n"); bad++; }
    /* summaries: status, completed, start, end */
    const uint32_t want[N * 4] = {1, 0, 0xFFFFFFFFu, 0xFFFFFFFFu, 4, 2, 1, 0, 5, 0, 1, 0, 0, 0, 0, 0};
    const uint8_t want_state[N] = {AFC_WORKFLOW_BUILT, AFC_WORKFLOW_BUILT, AFC_WORKFLOW_BUILT, AFC_WORKFLOW_HOST};
    for (int i = 0; i < N; i++) {
        if (state[i] != want_state[i]) { printf("workflow %d: state %d\n", i, state[i]); bad++; }
        if (memcmp(summary + 4 * i, want + 4 * i, 16) != 0) {
            printf("workflow %d: summary %u %u %u %u\n", i, summary[4 * i], summary[4 * i + 1], summary[4 * i + 2], summary[4 * i + 3]);
            bad++;
        }
    }
    if (doc_off[4] != doc_off[3]) { printf("a HOST workflow has a document\n"); bad++; }
    /* every built document verifies and ends in its proofValue */
    afc_keyset* ks = NULL;
    if (afc_keyset_new_named(ctx, pks, didbuf, did_off, K, &ks) != AFC_OK) { fprintf(stderr, "keyset\n"); return 5; }
    uint8_t status[N - 1];
    if (afc_vc_verify_stored_batch(ctx, ks, AFC_DOC_WORKFLOW_VC, docs, doc_off, N - 1, status, NULL) != AFC_OK) { fprintf(stderr, "verify\n"); return 6; }
    for (int i = 0; i < N - 1; i++) {
        if (status[i] != AFC_VC_VALID) { printf("document %d: status %d\n", i, status[i]); bad++; }
        const uint8_t* d = docs + doc_off[i];
        const uint64_t len = doc_off[i + 1] - doc_off[i];
        if (len < 90 || memcmp(d + len - 89, pv + 86 * i, 86) != 0 || memcmp(d + len - 3, "\"}}", 3) != 0) { printf("document %d: proofValue\n", i); bad++; }
    }
    {
        const char* arr = "\"componentVcIds\":[]";
        const size_t al = strlen(arr);
        int found = 0;
        for (uint64_t k = 0; k + al <= doc_off[1]; k++) found |= memcmp(docs + k, arr, al) == 0;
        if (!found) { printf("document 0: no empty array\n"); bad++; }
    }
    afc_keyset_free(ks);
    free(docs);
    afc_destroy(ctx);
    if (bad) return 1;
    printf("workflow_vc ok\n");
    return 0;
}
