/* tests/c_abi/json_vc.c — a plain-C caller of afc_vc_verify_json_batch (include/afcrypto.h), compiled as C99 with -pedantic against
 * the header alone, as cgo would: one execution VC pretty-printed as json.dumps(doc, indent=2) writes it, the same with one value
 * changed, and the same with two members swapped.
 * Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_vcjson_c_abi.py. */
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

int main(void) {
    afc_ctx* ctx = NULL;
    int rc = afc_init(0, &ctx);
    if (rc == AFC_ECUDA) { printf("no usable GPU: %s (the library has no CPU path)\n", afc_strerror(rc)); return 77; }
    if (rc != AFC_OK) { fprintf(stderr, "afc_init: %s\n", afc_strerror(rc)); return 2; }
    int bad = 0;
    /* tests/golden/go_cases.json, the first case, pretty-printed: the device re-marshals it to the bytes Go signed (VALID); with the
     * issuance date changed it does not verify (INVALID); with "id" and "issuer" swapped it is not the struct's member order, which
     * the caller's own Unmarshal -> Marshal -> Verify handles (HOST) */
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
        uint8_t vpk[32];
        unhex("00fabe35c569411ed5306ee09f41c8e9ce2817c50ee419fdb32923c5945e2ffc", vpk);
        const size_t L = sizeof(pretty) - 1;
        uint8_t* docs = (uint8_t*)malloc(3 * L);
        memcpy(docs, pretty, L);
        memcpy(docs + L, pretty, L);
        char* date = strstr((char*)docs + L, "\"issuanceDate\": \"2");
        date[17] = '3';                                                       /* 2026-... -> 3026-... */
        /* "id": "...",\n  "issuer": "..."  ->  "issuer": "...",\n  "id": "..." */
        {
            const char* id = strstr(pretty, "\"id\": ");
            const char* iss = strstr(pretty, "\"issuer\": ");
            const char* iss_end = strchr(iss, ',');
            const char* id_end = strchr(id, ',');
            size_t pre = (size_t)(id - pretty), n_id = (size_t)(id_end - id), n_gap = (size_t)(iss - id_end), n_iss = (size_t)(iss_end - iss);
            uint8_t* d = docs + 2 * L;
            memcpy(d, pretty, pre);
            memcpy(d + pre, iss, n_iss);
            memcpy(d + pre + n_iss, id_end, n_gap);
            memcpy(d + pre + n_iss + n_gap, id, n_id);
            memcpy(d + pre + n_iss + n_gap + n_id, iss_end, L - (size_t)(iss_end - pretty));
        }
        uint64_t doff[4] = {0, L, 2 * L, 3 * L}, did_off[2] = {0, strlen(did)};
        uint8_t vst[3] = {9, 9, 9};
        uint32_t vfields[12];
        afc_keyset* ks = NULL;
        rc = afc_keyset_new_named(ctx, vpk, (const uint8_t*)did, did_off, 1, &ks);
        if (rc) { fprintf(stderr, "keyset_new_named: %s\n", afc_strerror(rc)); return 3; }
        rc = afc_vc_verify_json_batch(ctx, ks, AFC_DOC_EXECUTION_VC, docs, doff, 3, vst, vfields);
        bad += rc != 0 || vst[0] != AFC_VC_VALID || vst[1] != AFC_VC_INVALID || vst[2] != AFC_VC_HOST;
        bad += vfields[1] != strlen(did) || memcmp(docs + vfields[0], did, strlen(did)) != 0;
        if (vst[0] != AFC_VC_VALID || vst[1] != AFC_VC_INVALID || vst[2] != AFC_VC_HOST) fprintf(stderr, "MISMATCH json VC statuses %d %d %d\n", vst[0], vst[1], vst[2]);
        afc_keyset_free(ks);
        free(docs);
    }
    afc_destroy(ctx);
    if (bad) { fprintf(stderr, "%d check(s) failed\n", bad); return 1; }
    printf("json_vc ok\n");
    return 0;
}
