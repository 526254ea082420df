/* tests/c_abi/stored_vc.c — a plain-C caller of the stored-document entry points of libafcrypto.so (include/afcrypto.h), compiled
 * as C99 with -pedantic against the header alone, as cgo would: afc_keyset_new_named + afc_vc_verify_stored_batch on one stored
 * execution VC, the same with one value changed, and the same with a space inserted.
 * Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_vcdoc_c_abi.py. */
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
    /* a stored execution VC (tests/golden/go_cases.json, the first case) verified from its bytes: as stored it verifies, with one
     * value changed it does not, with a space inserted it is left to the caller's own Unmarshal -> Marshal -> Verify (VCService.VerifyVC,
     * internal/services/vc_service.go:242-289) */
    {
        static const char stored[] =
    "{\"@context\":[\"https://www.w3.org/2018/credentials/v1\",\"https://agentfield.example.com/contexts/execution/v"
    "1\"],\"type\":[\"VerifiableCredential\",\"AgentFieldExecutionCredential\"],\"id\":\"urn:agentfield:vc:vc-178997"
    "1100759287000\",\"issuer\":\"did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A\",\"issuanceDate\":\"2026-"
    "09-21T06:00:00Z\",\"credentialSubject\":{\"executionId\":\"exec_0000\",\"workflowId\":\"wf_\\u003c0\\u003e\",\""
    "sessionId\":\"sess_0\",\"caller\":{\"did\":\"did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A\",\"type\""
    ":\"agent\",\"agentNodeDid\":\"did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A\"},\"target\":{\"did\":\""
    "\",\"agentNodeDid\":\"did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A\",\"functionName\":\"\"},\"execut"
    "ion\":{\"inputHash\":\"LcOQZrtCEWLLHIf8LxBLHqxeuQhh29gbI2UNPfFHENM\",\"outputHash\":\"dCNOmK_nSY-12vHzasLXiswzl"
    "GT5UHA7jAGYkvmCuQs\",\"timestamp\":\"2026-09-21T06:00:00Z\",\"durationMs\":782226,\"status\":\"succeeded\"},\"a"
    "udit\":{\"inputDataHash\":\"LcOQZrtCEWLLHIf8LxBLHqxeuQhh29gbI2UNPfFHENM\",\"outputDataHash\":\"dCNOmK_nSY-12vHz"
    "asLXiswzlGT5UHA7jAGYkvmCuQs\",\"metadata\":{\"agentfield_version\":\"1.0.0\",\"vc_version\":\"1.0\"}}},\"proof\""
    ":{\"type\":\"Ed25519Signature2020\",\"created\":\"2026-09-21T06:00:00Z\",\"verificationMethod\":\"did:key:z7QEA"
    "-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A#key-1\",\"proofPurpose\":\"assertionMethod\",\"proofValue\":\"rTWiLP"
    "EIrGYgjmmYZpPQIkw3bqD9dZJgXn7zQN6nruw5YBnynlt4PWvSJFTKxHsDZW90XrWb02haR6N-wq0qCg\"}}";
        const char* did = "did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A";
        uint8_t vpk[32];
        unhex("00fabe35c569411ed5306ee09f41c8e9ce2817c50ee419fdb32923c5945e2ffc", vpk);
        const size_t L = sizeof(stored) - 1;
        uint8_t* docs = (uint8_t*)malloc(3 * L + 1);
        memcpy(docs, stored, L);
        memcpy(docs + L, stored, L);
        char* date = strstr((char*)docs + L, "\"issuanceDate\":\"2");
        date[16] = '3';                                                       /* 2026-... -> 3026-...: still canonical */
        docs[2 * L] = '{'; docs[2 * L + 1] = ' ';
        memcpy(docs + 2 * L + 2, stored + 1, L - 1);                          /* { "@context":...: not the form Go writes */
        uint64_t doff[4] = {0, L, 2 * L, 3 * L + 1}, did_off[2] = {0, strlen(did)};
        uint8_t vst[3] = {9, 9, 9};
        uint32_t vfields[12];
        afc_keyset* ks = NULL;
        rc = afc_keyset_new_named(ctx, vpk, (const uint8_t*)did, did_off, 1, &ks);
        if (rc) { fprintf(stderr, "keyset_new_named: %s\n", afc_strerror(rc)); return 3; }
        rc = afc_vc_verify_stored_batch(ctx, ks, AFC_DOC_EXECUTION_VC, docs, doff, 3, vst, vfields);
        bad += rc != 0 || vst[0] != AFC_VC_VALID || vst[1] != AFC_VC_INVALID || vst[2] != AFC_VC_HOST;
        bad += vfields[1] != strlen(did) || memcmp(docs + vfields[0], did, strlen(did)) != 0;
        if (vst[0] != AFC_VC_VALID || vst[1] != AFC_VC_INVALID || vst[2] != AFC_VC_HOST) fprintf(stderr, "MISMATCH stored VC statuses %d %d %d\n", vst[0], vst[1], vst[2]);
        afc_keyset_free(ks);
        free(docs);
    }
    afc_destroy(ctx);
    if (bad) { fprintf(stderr, "%d check(s) failed\n", bad); return 1; }
    printf("stored_vc ok\n");
    return 0;
}
