/* tests/c_abi/did_reregister.c — a plain-C caller of afc_did_reregister_batch (include/afcrypto.h), compiled as C99 with -pedantic against
 * the header alone, as cgo would.  First, with no GPU needed: afc_did_reregister_bound is additive over requests and reads only the ends of
 * its offset arrays.  Then on the GPU: three known agents (nothing changed; one reasoner removed; a new reasoner next to a removed skill)
 * in one call, their states, counts, flags and key slot (equal to afc_ed25519_expand_batch of SHA-256(master || path)); every malformed
 * input is AFC_EINVAL; n = 0 writes body_off[0] = 0.
 * Exit code 0 = all good; 77 = no usable GPU (after the bound checks passed); anything else = a failed check.  Built and run by
 * tests/test_didrereg_c_abi.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "afcrypto.h"

#define N 3
#define M 5  /* request ids */
#define G 5  /* registered components */

static const char* agent_list[3 * N] = {"did:key:zA", "{\"x\":\"a\"}", "m/44'/1'/0'", "did:key:zB", "{\"x\":\"b\"}", "m/44'/1'/1'",
                                        "did:key:zC", "{ \"x\" : \"c\" }", "m/44'/1'/2'"};
/* agent 0: reasoner r0; agent 1: reasoners r0, r1; agent 2: skill s0, reasoner q */
static const char* reg_list[5 * G] = {"r0", "did:key:zR0", "{}", "m/44'/1'/0'/0'/0'", "r0",
                                      "r0", "did:key:zR1", "{}", "m/44'/1'/1'/0'/0'", "r0",
                                      "r1", "did:key:zR2", "{}", "m/44'/1'/1'/0'/1'", "",
                                      "q", "did:key:zQ", "{}", "m/44'/1'/2'/0'/0'", "q",
                                      "s0", "did:key:zS", "{}", "m/44'/1'/2'/1'/0'", "s0"};
static const uint64_t reg_idx[2 * N + 1] = {0, 1, 1, 3, 3, 4, 5};
static const char* id_list[M] = {"r0", "r1", "q", "new", "new"};     /* agent 0: r0; agent 1: r1; agent 2: q, new, new (no skills) */
static const uint64_t id_idx[2 * N + 1] = {0, 1, 1, 2, 2, 5, 5};

static void cat(const char* const* s, int k, uint8_t* buf, uint64_t* off) {
    int i;
    off[0] = 0;
    for (i = 0; i < k; i++) { memcpy(buf + off[i], s[i], strlen(s[i])); off[i + 1] = off[i] + strlen(s[i]); }
}

int main(void) {
    uint8_t agent_cols[512], reg_cols[512], ids[64];
    uint64_t agent_col_off[3 * N + 1], reg_col_off[5 * G + 1], id_off[M + 1];
    cat(agent_list, 3 * N, agent_cols, agent_col_off);
    cat(reg_list, 5 * G, reg_cols, reg_col_off);
    cat(id_list, M, ids, id_off);
    const char* server = "server-<1>";
    const uint64_t slen = strlen(server);
    int bad = 0, i;
    /* the bound: additive, and read only from the array ends */
    const uint64_t cap = afc_did_reregister_bound(agent_col_off, id_idx, id_off, reg_idx, reg_col_off, N, slen);
    {
        uint64_t sum = 0, ai[4], ii[3], io[M + 1], ri[3], ro[5 * G + 1];
        for (i = 0; i < N; i++) {     /* request i alone, through the same arrays' absolute offsets */
            ai[0] = agent_col_off[3 * i]; ai[3] = agent_col_off[3 * i + 3]; ai[1] = ai[2] = 0;
            ii[0] = id_idx[2 * i]; ii[2] = id_idx[2 * i + 2]; ii[1] = 0;
            ri[0] = reg_idx[2 * i]; ri[2] = reg_idx[2 * i + 2]; ri[1] = 0;
            sum += afc_did_reregister_bound(ai, ii, id_off, ri, reg_col_off, 1, slen);
        }
        if (cap == 0 || sum != cap) { fprintf(stderr, "bound not additive: %llu vs %llu\n", (unsigned long long)sum, (unsigned long long)cap); bad++; }
        memset(io, 0, sizeof io); io[0] = id_off[0]; io[M] = id_off[M];
        memset(ro, 0, sizeof ro); ro[0] = reg_col_off[0]; ro[5 * G] = reg_col_off[5 * G];
        {
            uint64_t ae[3 * N + 1];
            memset(ae, 0, sizeof ae); ae[0] = agent_col_off[0]; ae[3 * N] = agent_col_off[3 * N];
            if (afc_did_reregister_bound(ae, id_idx, io, reg_idx, ro, N, slen) != cap) { fprintf(stderr, "bound reads inner offsets\n"); bad++; }
        }
        if (afc_did_reregister_bound(agent_col_off, id_idx, id_off, reg_idx, reg_col_off, 0, slen) != 0) bad++;
        if (afc_did_reregister_bound(NULL, id_idx, id_off, reg_idx, reg_col_off, N, slen) != 0) bad++;
    }
    if (bad) { fprintf(stderr, "%d failed bound checks\n", bad); return 1; }
    printf("bound ok\n");
    afc_ctx* ctx = NULL;
    int rc = afc_init(0, &ctx);
    if (rc == AFC_ECUDA) { printf("no usable GPU: %s (the library has no CPU path)\n", afc_strerror(rc)); return 77; }
    if (rc != AFC_OK) { fprintf(stderr, "afc_init: %s\n", afc_strerror(rc)); return 2; }
    uint8_t master[32];
    for (i = 0; i < 32; i++) master[i] = (uint8_t)(i * 5 + 1);
    const uint32_t agent_index[N] = {0, 1, 2};
    uint8_t* body = malloc(cap);
    static uint8_t expanded[2 * N * 96], pks[2 * N * 32], dids[2 * N * AFC_DID_CHARS], paths[2 * N * AFC_DID_PATH_SLOT], state[N], reg_flags[G], id_flags[M];
    uint32_t counts[4 * N];
    uint64_t body_off[N + 1];
#define CALL(ms, aoff, iidx, ioff, ridx, roff, c, nn) \
    afc_did_reregister_batch(ctx, ms, (const uint8_t*)server, slen, agent_cols, aoff, agent_index, iidx, ids, ioff, ridx, reg_cols, roff, nn, state, \
                             counts, expanded, pks, dids, paths, reg_flags, id_flags, body, c, body_off)
    rc = CALL(master, agent_col_off, id_idx, id_off, reg_idx, reg_col_off, cap, N);
    if (rc != AFC_OK) { fprintf(stderr, "reregister: %s\n", afc_strerror(rc)); return 3; }
    if (state[0] != AFC_DIDRR_UNCHANGED || state[1] != AFC_DIDRR_REMOVED || state[2] != AFC_DIDRR_PARTIAL) { fprintf(stderr, "state\n"); bad++; }
    if (counts[4 * 1 + 2] != 1 || counts[4 * 2 + 0] != 1 || counts[4 * 2 + 3] != 1 || counts[4 * 2 + 1] != 0) { fprintf(stderr, "counts\n"); bad++; }
    if (reg_flags[0] || reg_flags[1] != AFC_DIDRR_GONE || reg_flags[2] || reg_flags[3] || reg_flags[4] != AFC_DIDRR_GONE) { fprintf(stderr, "reg_flags\n"); bad++; }
    if (id_flags[2] || id_flags[3] != AFC_DIDRR_NEW || id_flags[4] != (AFC_DIDRR_NEW | AFC_DID_KEPT)) { fprintf(stderr, "id_flags\n"); bad++; }
    /* agent 2's new reasoner: one survivor (q), so path index 1 */
    {
        uint8_t msg[80], seed[32], want[96];
        const size_t pl = strlen((const char*)paths + AFC_DID_PATH_SLOT * 4);
        uint64_t moff[2] = {0, 32 + pl};
        memcpy(msg, master, 32); memcpy(msg + 32, paths + AFC_DID_PATH_SLOT * 4, pl);
        if (pl < 20 || memcmp(paths + AFC_DID_PATH_SLOT * 4 + pl - 6, "/0'/1'", 6) != 0) { fprintf(stderr, "path index\n"); bad++; }
        if (afc_sha256_batch(ctx, msg, moff, 1, seed) != AFC_OK || afc_ed25519_expand_batch(ctx, seed, 1, want) != AFC_OK) return 4;
        if (memcmp(want, expanded + 4 * 96, 96) != 0 || memcmp(pks + 4 * 32, want + 64, 32) != 0) { fprintf(stderr, "key slot\n"); bad++; }
        if (memcmp(dids + AFC_DID_CHARS * 4, "did:key:z7", 10) != 0) { fprintf(stderr, "did\n"); bad++; }
        for (i = 0; i < 96; i++) if (expanded[i] || expanded[5 * 96 + i]) { fprintf(stderr, "unused slot\n"); bad++; break; }
        memset(seed, 0, sizeof seed); memset(want, 0, sizeof want);
    }
    for (i = 0; i < N; i++) {
        const char* b = (const char*)body + body_off[i];
        const size_t len = (size_t)(body_off[i + 1] - body_off[i]);
        if (len < 60 || strncmp(b, "{\"success\":true,\"identity_package\":{\"agent_did\":{\"did\":\"did:key:z", 62) != 0 || b[len - 1] != '}') {
            fprintf(stderr, "body %d\n", i); bad++;
        }
    }
    /* malformed inputs */
    if (CALL(NULL, agent_col_off, id_idx, id_off, reg_idx, reg_col_off, cap, N) != AFC_EINVAL) { fprintf(stderr, "null master\n"); bad++; }
    if (CALL(master, agent_col_off, id_idx, id_off, reg_idx, reg_col_off, cap - 1, N) != AFC_EINVAL) { fprintf(stderr, "cap\n"); bad++; }
    {
        uint64_t back[2 * N + 1], aoff[3 * N + 1], ioff[M + 1], roff[5 * G + 1];
        memcpy(back, id_idx, sizeof back); back[3] = 0;
        if (CALL(master, agent_col_off, back, id_off, reg_idx, reg_col_off, cap, N) != AFC_EINVAL) { fprintf(stderr, "id_idx\n"); bad++; }
        memcpy(back, reg_idx, sizeof back); back[3] = 0;
        if (CALL(master, agent_col_off, id_idx, id_off, back, reg_col_off, cap, N) != AFC_EINVAL) { fprintf(stderr, "reg_idx\n"); bad++; }
        memcpy(aoff, agent_col_off, sizeof aoff); aoff[2] = aoff[3] + 1;
        if (CALL(master, aoff, id_idx, id_off, reg_idx, reg_col_off, cap, N) != AFC_EINVAL) { fprintf(stderr, "agent_col_off\n"); bad++; }
        memcpy(ioff, id_off, sizeof ioff); ioff[1] = ioff[2] + 1;
        if (CALL(master, agent_col_off, id_idx, ioff, reg_idx, reg_col_off, cap, N) != AFC_EINVAL) { fprintf(stderr, "id_off\n"); bad++; }
        memcpy(roff, reg_col_off, sizeof roff); roff[7] = roff[8] + 1;
        if (CALL(master, agent_col_off, id_idx, id_off, reg_idx, roff, cap, N) != AFC_EINVAL) { fprintf(stderr, "reg_col_off\n"); bad++; }
        if (afc_did_reregister_batch(ctx, master, (const uint8_t*)server, slen, agent_cols, agent_col_off, agent_index, id_idx, ids, id_off, reg_idx,
                                     reg_cols, reg_col_off, N, state, counts, expanded, pks, dids, paths, NULL, id_flags, body, cap, body_off) != AFC_EINVAL) {
            fprintf(stderr, "null reg_flags\n"); bad++;
        }
        if (afc_did_reregister_batch(ctx, master, (const uint8_t*)server, slen, agent_cols, agent_col_off, agent_index, id_idx, ids, id_off, reg_idx,
                                     NULL, reg_col_off, N, state, counts, expanded, pks, dids, paths, reg_flags, id_flags, body, cap, body_off) != AFC_EINVAL) {
            fprintf(stderr, "null reg_cols\n"); bad++;
        }
    }
    body_off[0] = 7;
    if (CALL(master, agent_col_off, id_idx, id_off, reg_idx, reg_col_off, 0, 0) != AFC_OK || body_off[0] != 0) { fprintf(stderr, "n = 0\n"); bad++; }
    memset(expanded, 0, sizeof expanded);
    memset(body, 0, cap);
    free(body);
    afc_destroy(ctx);
    if (bad) { fprintf(stderr, "%d failed checks\n", bad); return 1; }
    printf("did_reregister ok\n");
    return 0;
}
