/* tests/c_abi/verify_request.c — a plain-C caller of afc_vc_verify_request_batch (include/afcrypto.h), compiled as C99 with -pedantic against
 * the header alone, as cgo would: four raw request bodies of POST /api/v1/did/verify — an execution VC pretty-printed inside
 * {"vc_document": ...} (200, valid), the same with its issuance date changed (200, invalid signature), a body that is an array (400) and a
 * vc_document that is a string (left to the caller).
 * Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_vcreq_c_abi.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "afcrypto.h"

static int unhex(const char* s, uint8_t* out) {
    int n = 0;
    for (; s[0] && s[1]; s += 2, n++) { unsigned v; if (sscanf(s, "%2x", &v) != 1) return -1; out[n] = (uint8_t)v; }
    return n;
}

static int same(const uint8_t* bodies, const uint64_t* off, int i, const char* want) {
    const size_t n = strlen(want);
    if (off[i + 1] - off[i] != n || memcmp(bodies + off[i], want, n) != 0) {
        fprintf(stderr, "MISMATCH body %d: %.*s\n", i, (int)(off[i + 1] - off[i]), (const char*)bodies + off[i]);
        return 1;
    }
    return 0;
}

int main(void) {
    afc_ctx* ctx = NULL;
    int rc = afc_init(0, &ctx);
    if (rc == AFC_ECUDA) { printf("no usable GPU: %s (the library has no CPU path)\n", afc_strerror(rc)); return 77; }
    if (rc != AFC_OK) { fprintf(stderr, "afc_init: %s\n", afc_strerror(rc)); return 2; }
    int bad = 0;
    /* tests/golden/go_cases.json, the first case, pretty-printed as json.dumps(doc, indent=2) writes it */
    {
        static const char pretty[] =
    "{\n  \"@context\": [\n    \"https://www.w3.org/2018/credentials/v1\",\n    \"https://agentfield.example.com/co"
    "ntexts/execution/v1\"\n  ],\n  \"type\": [\n    \"VerifiableCredential\",\n    \"AgentFieldExecutionCredential"
    "\"\n  ],\n  \"id\": \"urn:agentfield:vc:vc-1789971100759287000\",\n  \"issuer\": \"did:key:z7QEA-r41xWlBHtUwbu"
    "CfQcjpzigXxQ7kGf2zKSPFlF4v_A\",\n  \"issuanceDate\": \"2026-09-21T06:00:00Z\",\n  \"credentialSubject\": {\n  "
    "  \"executionId\": \"exec_0000\",\n    \"workflowId\": \"wf_<0>\",\n    \"sessionId\": \"sess_0\",\n    \"call"
    "er\": {\n      \"did\": \"did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A\",\n      \"type\": \"agent\""
    ",\n      \"agentNodeDid\": \"did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A\"\n    },\n    \"target\""
    ": {\n      \"did\": \"\",\n      \"agentNodeDid\": \"did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A\""
    ",\n      \"functionName\": \"\"\n    },\n    \"execution\": {\n      \"inputHash\": \"LcOQZrtCEWLLHIf8LxBLHqxe"
    "uQhh29gbI2UNPfFHENM\",\n      \"outputHash\": \"dCNOmK_nSY-12vHzasLXiswzlGT5UHA7jAGYkvmCuQs\",\n      \"timest"
    "amp\": \"2026-09-21T06:00:00Z\",\n      \"durationMs\": 782226,\n      \"status\": \"succeeded\"\n    },\n    "
    "\"audit\": {\n      \"inputDataHash\": \"LcOQZrtCEWLLHIf8LxBLHqxeuQhh29gbI2UNPfFHENM\",\n      \"outputDataHas"
    "h\": \"dCNOmK_nSY-12vHzasLXiswzlGT5UHA7jAGYkvmCuQs\",\n      \"metadata\": {\n        \"agentfield_version\": "
    "\"1.0.0\",\n        \"vc_version\": \"1.0\"\n      }\n    }\n  },\n  \"proof\": {\n    \"type\": \"Ed25519Sign"
    "ature2020\",\n    \"created\": \"2026-09-21T06:00:00Z\",\n    \"verificationMethod\": \"did:key:z7QEA-r41xWlBH"
    "tUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A#key-1\",\n    \"proofPurpose\": \"assertionMethod\",\n    \"proofValue\": \""
    "rTWiLPEIrGYgjmmYZpPQIkw3bqD9dZJgXn7zQN6nruw5YBnynlt4PWvSJFTKxHsDZW90XrWb02haR6N-wq0qCg\"\n  }\n}";
        const char* did = "did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A";
        const char* head = "{\"vc_document\": ";
        const char* array = "[]";
        const char* str = "{\"vc_document\":\"x\"}";
        uint8_t vpk[32];
        unhex("00fabe35c569411ed5306ee09f41c8e9ce2817c50ee419fdb32923c5945e2ffc", vpk);
        const size_t L = strlen(head) + sizeof(pretty) - 1 + 1;
        uint8_t* reqs = (uint8_t*)malloc(2 * L + strlen(array) + strlen(str));
        uint64_t roff[5];
        roff[0] = 0;
        for (int k = 0; k < 2; k++) {
            uint8_t* r = reqs + k * L;
            memcpy(r, head, strlen(head));
            memcpy(r + strlen(head), pretty, sizeof(pretty) - 1);
            r[L - 1] = '}';
            roff[k + 1] = (uint64_t)(k + 1) * L;
        }
        char* date = strstr((char*)reqs + L, "\"issuanceDate\": \"2");
        date[17] = '3';                                                       /* 2026-... -> 3026-... */
        memcpy(reqs + 2 * L, array, strlen(array));
        roff[3] = roff[2] + strlen(array);
        memcpy(reqs + roff[3], str, strlen(str));
        roff[4] = roff[3] + strlen(str);
        uint64_t did_off[2] = {0, strlen(did)};
        afc_keyset* ks = NULL;
        rc = afc_keyset_new_named(ctx, vpk, (const uint8_t*)did, did_off, 1, &ks);
        if (rc) { fprintf(stderr, "keyset_new_named: %s\n", afc_strerror(rc)); return 3; }
        const uint64_t cap = afc_vc_verify_request_bound(roff, 4);
        uint8_t* bodies = (uint8_t*)malloc(cap);
        uint64_t boff[5];
        uint8_t st[4] = {9, 9, 9, 9};
        bad += afc_vc_verify_request_batch(ctx, ks, reqs, roff, 4, bodies, cap - 1, boff, st) != AFC_EINVAL;
        rc = afc_vc_verify_request_batch(ctx, ks, reqs, roff, 4, bodies, cap, boff, st);
        bad += rc != 0 || st[0] != AFC_VREQ_OK || st[1] != AFC_VREQ_OK || st[2] != AFC_VREQ_BAD_REQUEST || st[3] != AFC_VREQ_HOST;
        if (rc || st[0] || st[1] || st[2] != 1 || st[3] != 2) fprintf(stderr, "MISMATCH rc %d states %d %d %d %d\n", rc, st[0], st[1], st[2], st[3]);
        if (rc == 0) {
            bad += same(bodies, boff, 0, "{\"valid\":true,\"issuer_did\":\"did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A\","
                                         "\"issued_at\":\"2026-09-21T06:00:00Z\",\"message\":\"VC verified successfully\"}");
            bad += same(bodies, boff, 1, "{\"valid\":false,\"message\":\"Invalid signature\"}");
            bad += same(bodies, boff, 2, "{\"error\":\"Invalid request body\"}");
            bad += same(bodies, boff, 3, "");
        }
        afc_keyset_free(ks);
        free(bodies);
        free(reqs);
    }
    afc_destroy(ctx);
    if (bad) { fprintf(stderr, "%d check(s) failed\n", bad); return 1; }
    printf("verify_request ok\n");
    return 0;
}
