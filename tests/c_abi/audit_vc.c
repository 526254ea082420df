/* tests/c_abi/audit_vc.c — a plain-C caller of the audit entry point of libafcrypto.so (include/afcrypto.h), compiled as C99 with
 * -pedantic against the header alone, as cgo would: afc_vc_audit_stored_batch on one stored execution VC against its record, against
 * the record with one column changed and with the status spelled differently, and the document with a space inserted; then the
 * argument errors.  Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_audit_c_abi.py. */
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

/* packs the AFC_AUDIT_COLUMNS values of each of n records into cols / col_off */
static void pack_columns(const char* const* vals, uint32_t n, uint8_t* cols, uint64_t* col_off) {
    uint64_t at = 0;
    uint32_t k;
    col_off[0] = 0;
    for (k = 0; k < n * AFC_AUDIT_COLUMNS; k++) {
        size_t l = strlen(vals[k]);
        memcpy(cols + at, vals[k], l);
        at += l;
        col_off[k + 1] = at;
    }
}

int main(void) {
    afc_ctx* ctx = NULL;
    int rc = afc_init(0, &ctx);
    if (rc == AFC_ECUDA) { printf("no usable GPU: %s (the library has no CPU path)\n", afc_strerror(rc)); return 77; }
    if (rc != AFC_OK) { fprintf(stderr, "afc_init: %s\n", afc_strerror(rc)); return 2; }
    int bad = 0;
    {
        /* tests/golden/go_cases.json, the first case, and the ExecutionVC record stored with it (its workflowId is written with
         * \u003c / \u003e escapes: the record holds the unescaped text) */
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
        const char* pv = "rTWiLPEIrGYgjmmYZpPQIkw3bqD9dZJgXn7zQN6nruw5YBnynlt4PWvSJFTKxHsDZW90XrWb02haR6N-wq0qCg";
        const char* ih = "LcOQZrtCEWLLHIf8LxBLHqxeuQhh29gbI2UNPfFHENM";
        const char* oh = "dCNOmK_nSY-12vHzasLXiswzlGT5UHA7jAGYkvmCuQs";
        const char* vals[4 * AFC_AUDIT_COLUMNS] = {
            did, "exec_0000", "wf_<0>", "sess_0", did, "", "succeeded", ih, oh, pv,          /* as stored */
            did, "exec_0000", "wf_<1>", "sess_0", did, "", "succeeded", ih, oh, pv,          /* workflow_id changed */
            did, "exec_0000", "wf_<0>", "sess_0", did, "", " Completed ", ih, oh, pv,        /* the same status, spelled differently */
            did, "exec_0000", "wf_<0>", "sess_0", did, "", "succeeded", ih, oh, pv};         /* (the document is not canonical) */
        uint8_t vpk[32];
        unhex("00fabe35c569411ed5306ee09f41c8e9ce2817c50ee419fdb32923c5945e2ffc", vpk);
        const size_t L = sizeof(stored) - 1;
        uint8_t* docs = (uint8_t*)malloc(4 * L + 1);
        uint8_t* cols = (uint8_t*)malloc(4096);
        uint64_t col_off[4 * AFC_AUDIT_COLUMNS + 1];
        memcpy(docs, stored, L);
        memcpy(docs + L, stored, L);
        memcpy(docs + 2 * L, stored, L);
        docs[3 * L] = '{'; docs[3 * L + 1] = ' ';
        memcpy(docs + 3 * L + 2, stored + 1, L - 1);
        uint64_t doff[5] = {0, L, 2 * L, 3 * L, 4 * L + 1}, did_off[2] = {0, strlen(did)};
        uint8_t st[4] = {9, 9, 9, 9};
        uint32_t iss[4] = {7, 7, 7, 7};
        afc_keyset* ks = NULL;
        pack_columns(vals, 4, cols, col_off);
        rc = afc_keyset_new_named(ctx, vpk, (const uint8_t*)did, did_off, 1, &ks);
        if (rc) { fprintf(stderr, "keyset_new_named: %s\n", afc_strerror(rc)); return 3; }
        rc = afc_vc_audit_stored_batch(ctx, ks, AFC_DOC_EXECUTION_VC, docs, doff, cols, col_off, 4, st, iss);
        bad += rc != 0 || st[0] != AFC_VC_VALID || st[1] != AFC_VC_VALID || st[2] != AFC_VC_VALID || st[3] != AFC_VC_HOST;
        bad += iss[0] != 0 || iss[1] != AFC_AUDIT_WORKFLOW_ID_MISMATCH || iss[2] != 0 || iss[3] != 0;
        if (bad) fprintf(stderr, "MISMATCH audit rc %d statuses %d %d %d %d issues %u %u %u %u\n", rc, st[0], st[1], st[2], st[3], iss[0], iss[1], iss[2], iss[3]);
        /* argument errors: an execution batch needs its columns, a workflow batch takes none, the key set must be named */
        bad += afc_vc_audit_stored_batch(ctx, ks, AFC_DOC_EXECUTION_VC, docs, doff, NULL, NULL, 4, st, iss) != AFC_EINVAL;
        bad += afc_vc_audit_stored_batch(ctx, ks, AFC_DOC_WORKFLOW_VC, docs, doff, cols, col_off, 4, st, iss) != AFC_EINVAL;
        bad += afc_vc_audit_stored_batch(ctx, ks, 7, docs, doff, cols, col_off, 4, st, iss) != AFC_EINVAL;
        afc_keyset_free(ks);
        ks = NULL;
        rc = afc_keyset_new(ctx, vpk, 1, &ks);
        bad += rc != 0 || afc_vc_audit_stored_batch(ctx, ks, AFC_DOC_EXECUTION_VC, docs, doff, cols, col_off, 4, st, iss) != AFC_ESTATE;
        afc_keyset_free(ks);
        free(docs);
        free(cols);
    }
    afc_destroy(ctx);
    if (bad) { fprintf(stderr, "%d check(s) failed\n", bad); return 1; }
    printf("audit_vc ok\n");
    return 0;
}
