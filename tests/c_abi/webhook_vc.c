/* tests/c_abi/webhook_vc.c — a plain-C caller of afc_webhook_sign_batch (include/afcrypto.h), compiled as C99 with -pedantic against
 * the header alone, as cgo would: three deliveries (a completed one whose result is re-marshalled, a failed one with an error
 * message, one whose status is not printable ASCII) in one call.  The bodies must be the expected bytes, the header must equal
 * afc_hmac_sha256_batch of the body written as "sha256=" + hex, and the third delivery must be AFC_WEBHOOK_HOST with a zero-length body.
 * Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_webhook_c_abi.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "afcrypto.h"

#define N 3

int main(void) {
    afc_ctx* ctx = NULL;
    int rc = afc_init(0, &ctx);
    if (rc == AFC_ECUDA) { printf("no usable GPU: %s (the library has no CPU path)\n", afc_strerror(rc)); return 77; }
    if (rc != AFC_OK) { fprintf(stderr, "afc_init: %s\n", afc_strerror(rc)); return 2; }
    const char* cols[N][AFC_WEBHOOK_COLUMNS] = {
        {"exec_1", "run_1", "succeeded", "node", "summarise", "reasoner", "2026-09-21T06:30:00Z", ""},
        {"exec_2", "run_<2>", "failed", "node", "rank", "skill", "2026-09-21T06:30:01Z", "boom & \"quoted\""},
        {"exec_3", "run_3", "done\xc2\xa0", "node", "f", "reasoner", "2026-09-21T06:30:02Z", ""},
    };
    const char* expect[N] = {
        "{\"event\":\"execution.completed\",\"execution_id\":\"exec_1\",\"workflow_id\":\"run_1\",\"status\":\"succeeded\",\"target\":\"node.summarise\","
        "\"type\":\"reasoner\",\"duration_ms\":1500,\"result\":{\"a\":[100000000000000000000,1.5,\"\\u003cb\\u003e\"],\"z\":null},"
        "\"timestamp\":\"2026-09-21T06:30:00Z\"}",
        "{\"event\":\"execution.failed\",\"execution_id\":\"exec_2\",\"workflow_id\":\"run_\\u003c2\\u003e\",\"status\":\"failed\",\"target\":\"node.rank\","
        "\"type\":\"skill\",\"error_message\":\"boom \\u0026 \\\"quoted\\\"\",\"timestamp\":\"2026-09-21T06:30:01Z\"}",
        "",
    };
    const char* results[N] = {"{\"z\": null, \"a\": [1e20, 1.50, \"<b>\"]}", "", "1"};
    const char* secret = "whsec_example";
    uint8_t colbuf[1024], resbuf[256], secbuf[64];
    uint64_t col_off[N * AFC_WEBHOOK_COLUMNS + 1], res_off[N + 1];
    uint32_t sec_off[N + 1];
    int64_t dur[N] = {1500, 0, 7};
    uint8_t flags[N] = {AFC_WEBHOOK_HAS_DURATION | AFC_WEBHOOK_HAS_SECRET, AFC_WEBHOOK_HAS_ERROR_MESSAGE, AFC_WEBHOOK_HAS_SECRET};
    size_t at = 0, ra = 0, sa = 0;
    int i, k;
    for (i = 0; i < N; i++) {
        for (k = 0; k < AFC_WEBHOOK_COLUMNS; k++) {
            col_off[i * AFC_WEBHOOK_COLUMNS + k] = at;
            memcpy(colbuf + at, cols[i][k], strlen(cols[i][k])); at += strlen(cols[i][k]);
        }
        res_off[i] = ra; memcpy(resbuf + ra, results[i], strlen(results[i])); ra += strlen(results[i]);
        sec_off[i] = (uint32_t)sa;
        if (flags[i] & AFC_WEBHOOK_HAS_SECRET) { memcpy(secbuf + sa, secret, strlen(secret)); sa += strlen(secret); }
    }
    col_off[N * AFC_WEBHOOK_COLUMNS] = at; res_off[N] = ra; sec_off[N] = (uint32_t)sa;
    const uint64_t cap = afc_webhook_bound(col_off, res_off, N);
    uint8_t* bodies = (uint8_t*)malloc(cap);
    uint64_t body_off[N + 1];
    uint8_t headers[N][AFC_WEBHOOK_HEADER_CHARS], status[N];
    if (afc_webhook_sign_batch(ctx, colbuf, col_off, dur, flags, resbuf, res_off, secbuf, sec_off, N, bodies, cap - 1, body_off, &headers[0][0], status)
        != AFC_EINVAL) { fprintf(stderr, "a buffer below the bound must be AFC_EINVAL\n"); return 3; }
    rc = afc_webhook_sign_batch(ctx, colbuf, col_off, dur, flags, resbuf, res_off, secbuf, sec_off, N, bodies, cap, body_off, &headers[0][0], status);
    if (rc != AFC_OK) { fprintf(stderr, "afc_webhook_sign_batch: %s %s\n", afc_strerror(rc), afc_last_cuda_error(ctx)); return 4; }
    for (i = 0; i < N; i++) {
        const uint64_t len = body_off[i + 1] - body_off[i];
        if (len != strlen(expect[i]) || memcmp(bodies + body_off[i], expect[i], len)) {
            fprintf(stderr, "body %d: %.*s\n", i, (int)len, (const char*)bodies + body_off[i]); return 5;
        }
        if (status[i] != (i == 2 ? AFC_WEBHOOK_HOST : AFC_WEBHOOK_BUILT)) { fprintf(stderr, "status %d = %d\n", i, status[i]); return 6; }
    }
    {   /* the header of delivery 0 is the HMAC of its body */
        uint8_t tag[32];
        uint64_t off[2] = {0, body_off[1] - body_off[0]};
        uint32_t koff[2] = {0, (uint32_t)strlen(secret)};
        char want[AFC_WEBHOOK_HEADER_CHARS + 1];
        if (afc_hmac_sha256_batch(ctx, (const uint8_t*)secret, koff, bodies + body_off[0], off, 1, tag) != AFC_OK) return 7;
        memcpy(want, "sha256=", 7);
        for (k = 0; k < 32; k++) sprintf(want + 7 + 2 * k, "%02x", tag[k]);
        if (memcmp(headers[0], want, AFC_WEBHOOK_HEADER_CHARS)) { fprintf(stderr, "header 0 differs\n"); return 8; }
        for (k = 0; k < AFC_WEBHOOK_HEADER_CHARS; k++) if (headers[1][k] || headers[2][k]) { fprintf(stderr, "headers 1, 2 must be zero\n"); return 9; }
    }
    free(bodies);
    afc_destroy(ctx);
    printf("webhook_vc ok\n");
    return 0;
}
