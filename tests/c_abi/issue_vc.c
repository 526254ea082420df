/* tests/c_abi/issue_vc.c — a plain-C caller of afc_vc_issue_execution_batch (include/afcrypto.h), compiled as C99 with -pedantic
 * against the header alone, as cgo would: three issuers, four requests (nil, empty and 100-byte payloads, an error message that needs
 * escaping), issued in one call.  Every document must verify through afc_vc_verify_stored_batch, and every hash must equal
 * afc_sha256_batch of the payload's JSON text ("<std base64>" or null) written as base64url.
 * Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_vcissue_c_abi.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "afcrypto.h"

static size_t b64(const uint8_t* in, size_t n, char* out, int url) {
    const char* a = url ? "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789-_"
                        : "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    size_t o = 0, i;
    for (i = 0; i + 3 <= n; i += 3) {
        uint32_t v = (uint32_t)in[i] << 16 | (uint32_t)in[i + 1] << 8 | in[i + 2];
        out[o++] = a[v >> 18]; out[o++] = a[(v >> 12) & 63]; out[o++] = a[(v >> 6) & 63]; out[o++] = a[v & 63];
    }
    if (n - i == 1) {
        uint32_t v = (uint32_t)in[i] << 16;
        out[o++] = a[v >> 18]; out[o++] = a[(v >> 12) & 63];
        if (!url) { out[o++] = '='; out[o++] = '='; }
    } else if (n - i == 2) {
        uint32_t v = (uint32_t)in[i] << 16 | (uint32_t)in[i + 1] << 8;
        out[o++] = a[v >> 18]; out[o++] = a[(v >> 12) & 63]; out[o++] = a[(v >> 6) & 63];
        if (!url) out[o++] = '=';
    }
    return o;
}

#define N 4
#define K 3

int main(void) {
    afc_ctx* ctx = NULL;
    int rc = afc_init(0, &ctx);
    if (rc == AFC_ECUDA) { printf("no usable GPU: %s (the library has no CPU path)\n", afc_strerror(rc)); return 77; }
    if (rc != AFC_OK) { fprintf(stderr, "afc_init: %s\n", afc_strerror(rc)); return 2; }
    int bad = 0;
    uint8_t seeds[K * 32], exp[K * 96], pks[K * 32];
    for (int i = 0; i < K * 32; i++) seeds[i] = (uint8_t)(i * 7 + 3);
    if (afc_ed25519_expand_batch(ctx, seeds, K, exp) != AFC_OK) { fprintf(stderr, "expand\n"); return 3; }
    char dids[K][64];
    uint8_t didbuf[K * 64];
    uint64_t did_off[K + 1] = {0};
    for (int k = 0; k < K; k++) {
        uint8_t raw[34] = {0xed, 0x01};
        memcpy(pks + 32 * k, exp + 96 * k + 64, 32);
        memcpy(raw + 2, pks + 32 * k, 32);
        strcpy(dids[k], "did:key:z");
        dids[k][9 + b64(raw, 34, dids[k] + 9, 1)] = 0;
        memcpy(didbuf + did_off[k], dids[k], strlen(dids[k]));
        did_off[k + 1] = did_off[k] + strlen(dids[k]);
    }
    /* the columns, AFC_ISSUE_COLUMNS per request */
    const char* err = "tool <fetch> failed & \"retried\"\n";
    const char* col[N][AFC_ISSUE_COLUMNS];
    uint32_t ki[N];
    int64_t dur[N] = {0, 1234, -5, 86400000};
    for (int i = 0; i < N; i++) {
        ki[i] = (uint32_t)(i % K);
        const char* c[AFC_ISSUE_COLUMNS] = {"vc-1", dids[i % K], "2026-09-21T06:00:00Z", "exec_1", "wf_1", "sess_1", "agent", dids[(i + 1) % K],
                                            "", "summarize", "2026-09-21T06:00:00Z", "succeeded", i == 2 ? err : "", "2026-09-21T06:00:01Z"};
        memcpy(col[i], c, sizeof c);
    }
    static uint8_t cols[8192];
    uint64_t col_off[N * AFC_ISSUE_COLUMNS + 1] = {0};
    for (int j = 0; j < N * AFC_ISSUE_COLUMNS; j++) {
        const char* s = col[j / AFC_ISSUE_COLUMNS][j % AFC_ISSUE_COLUMNS];
        memcpy(cols + col_off[j], s, strlen(s));
        col_off[j + 1] = col_off[j] + strlen(s);
    }
    /* payloads: input i then output i; 0: nil / empty, 1: "hello" / 100 bytes, 2: nil / nil, 3: 100 bytes / "hello" */
    static uint8_t pay[256];
    uint64_t pay_off[2 * N + 1] = {0};
    uint8_t nil[2 * N] = {1, 0, 0, 0, 1, 1, 0, 0};
    uint64_t plen[2 * N] = {0, 0, 5, 100, 0, 0, 100, 5};
    for (int j = 0; j < 2 * N; j++) pay_off[j + 1] = pay_off[j] + plen[j];
    for (uint64_t b = 0; b < pay_off[2 * N]; b++) pay[b] = (uint8_t)(b * 31 + 1);
    memcpy(pay + pay_off[2], "hello", 5);
    const uint64_t cap = afc_vc_issue_bound(col_off, N);
    uint8_t* docs = (uint8_t*)malloc(cap);
    uint64_t doc_off[N + 1];
    uint8_t hashes[N * 86], pv[N * 86];
    rc = afc_vc_issue_execution_batch(ctx, exp, K, ki, cols, col_off, dur, pay, pay_off, nil, AFC_ISSUE_HASH_DATA, N, NULL, docs, cap, doc_off,
                                      hashes, pv);
    if (rc != AFC_OK) { fprintf(stderr, "issue: %s\n", afc_strerror(rc)); return 4; }
    if (afc_vc_issue_execution_batch(ctx, exp, K, ki, cols, col_off, dur, pay, pay_off, nil, AFC_ISSUE_HASH_DATA, N, NULL, docs, cap - 1, doc_off,
                                     hashes, pv) != AFC_EINVAL) { printf("bound not enforced\n"); bad++; }
    /* every document verifies */
    afc_keyset* ks = NULL;
    if (afc_keyset_new_named(ctx, pks, didbuf, did_off, K, &ks) != AFC_OK) { fprintf(stderr, "keyset\n"); return 5; }
    uint8_t status[N];
    if (afc_vc_verify_stored_batch(ctx, ks, AFC_DOC_EXECUTION_VC, docs, doc_off, N, status, NULL) != AFC_OK) { fprintf(stderr, "verify\n"); return 6; }
    for (int i = 0; i < N; i++) {
        if (status[i] != AFC_VC_VALID) { printf("document %d: status %d\n", i, status[i]); bad++; }
        const uint8_t* d = docs + doc_off[i];
        const uint64_t len = doc_off[i + 1] - doc_off[i];
        if (len < 90 || memcmp(d + len - 89, pv + 86 * i, 86) != 0 || memcmp(d + len - 3, "\"}}", 3) != 0) { printf("document %d: proofValue\n", i); bad++; }
    }
    /* every hash is SHA-256 of the payload's JSON text, base64url */
    static uint8_t text[2048];
    uint64_t text_off[2 * N + 1] = {0};
    for (int j = 0; j < 2 * N; j++) {
        uint8_t* t = text + text_off[j];
        size_t m;
        if (nil[j]) { memcpy(t, "null", 4); m = 4; }
        else { t[0] = '"'; m = 1 + b64(pay + pay_off[j], (size_t)plen[j], (char*)t + 1, 0); t[m++] = '"'; }
        text_off[j + 1] = text_off[j] + m;
    }
    uint8_t dig[2 * N * 32];
    if (afc_sha256_batch(ctx, text, text_off, 2 * N, dig) != AFC_OK) { fprintf(stderr, "sha256\n"); return 7; }
    for (int j = 0; j < 2 * N; j++) {
        char want[44];
        b64(dig + 32 * j, 32, want, 1);
        if (memcmp(want, hashes + 43 * j, 43) != 0) { printf("hash %d differs\n", j); bad++; }
    }
    afc_keyset_free(ks);
    free(docs);
    afc_destroy(ctx);
    if (bad) return 1;
    printf("issue_vc ok\n");
    return 0;
}
