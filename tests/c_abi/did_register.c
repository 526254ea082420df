/* tests/c_abi/did_register.c — a plain-C caller of afc_did_register_batch (include/afcrypto.h), compiled as C99 with -pedantic against the
 * header alone, as cgo would: three agents (no components; two reasoners, an empty id and a repeated skill; an id that needs escaping)
 * registered in one call.  Each component's key must equal afc_ed25519_expand_batch of SHA-256(master || path) (afc_sha256_batch), its DID
 * must be did:key:z..., and the bodies must frame as the response does.  Argument errors must be AFC_EINVAL.
 * Exit code 0 = all good; 77 = no usable GPU; anything else = a failed check.  Built and run by tests/test_didreg_c_abi.py. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "afcrypto.h"

/* whether the n bytes at p (not NUL-terminated) hold the text s */
static int contains(const uint8_t* p, size_t n, const char* s) {
    const size_t k = strlen(s);
    size_t i;
    for (i = 0; i + k <= n; i++) if (memcmp(p + i, s, k) == 0) return 1;
    return 0;
}

#define N 3
#define M 6

int main(void) {
    afc_ctx* ctx = NULL;
    int rc = afc_init(0, &ctx);
    if (rc == AFC_ECUDA) { printf("no usable GPU: %s (the library has no CPU path)\n", afc_strerror(rc)); return 77; }
    if (rc != AFC_OK) { fprintf(stderr, "afc_init: %s\n", afc_strerror(rc)); return 2; }
    int bad = 0, i, c;
    uint8_t master[32];
    for (i = 0; i < 32; i++) master[i] = (uint8_t)(i * 7 + 3);
    const char* server = "server-<1>";
    const char* node_list[N] = {"bare", "agent-two", "agent\"three"};
    const char* id_list[M] = {"summarize", "", "translate", "tag", "tag", "a<b>&c"};
    const uint64_t id_idx[2 * N + 1] = {0, 0, 0, 3, 5, 6, 6};     /* bare: none; two: 3 reasoners, 2 skills; three: 1 reasoner */
    const uint32_t agent_index[N] = {0, 1, 2};
    uint8_t nodes[256], ids[256];
    uint64_t node_off[N + 1] = {0}, id_off[M + 1] = {0};
    for (i = 0; i < N; i++) { memcpy(nodes + node_off[i], node_list[i], strlen(node_list[i])); node_off[i + 1] = node_off[i] + strlen(node_list[i]); }
    for (i = 0; i < M; i++) { memcpy(ids + id_off[i], id_list[i], strlen(id_list[i])); id_off[i + 1] = id_off[i] + strlen(id_list[i]); }
    const uint64_t cap = afc_did_register_bound(node_off, id_idx, id_off, N, strlen(server));
    uint8_t* body = malloc(cap);
    static uint8_t expanded[(N + M) * 96], pks[(N + M) * 32], dids[(N + M) * AFC_DID_CHARS], paths[(N + M) * AFC_DID_PATH_SLOT], flags[N + M];
    uint64_t comp_off[N + 1], body_off[N + 1];
    rc = afc_did_register_batch(ctx, master, (const uint8_t*)server, strlen(server), nodes, node_off, agent_index, id_idx, ids, id_off, N, comp_off,
                                expanded, pks, dids, paths, flags, body, cap, body_off);
    if (rc != AFC_OK) { fprintf(stderr, "register: %s\n", afc_strerror(rc)); return 3; }
    /* components: bare 1; two: agent + summarize, translate + tag, tag (the first shadowed); three: agent + a<b>&c */
    if (comp_off[0] != 0 || comp_off[1] != 1 || comp_off[2] != 6 || comp_off[3] != 8) { fprintf(stderr, "comp_off\n"); bad++; }
    if (flags[4] != 0 || flags[5] != AFC_DID_KEPT || flags[0] != AFC_DID_KEPT) { fprintf(stderr, "flags\n"); bad++; }
    /* keys: SHA-256(master || path) through the library's own hash, then the expansion */
    const int C = (int)comp_off[N];
    uint8_t msgs[8 * 80], seeds[8 * 32], want[8 * 96];
    uint64_t moff[9] = {0};
    for (c = 0; c < C; c++) {
        const size_t pl = strlen((const char*)paths + AFC_DID_PATH_SLOT * c);
        memcpy(msgs + moff[c], master, 32);
        memcpy(msgs + moff[c] + 32, paths + AFC_DID_PATH_SLOT * c, pl);
        moff[c + 1] = moff[c] + 32 + pl;
    }
    if (afc_sha256_batch(ctx, msgs, moff, (uint32_t)C, seeds) != AFC_OK || afc_ed25519_expand_batch(ctx, seeds, (uint32_t)C, want) != AFC_OK) return 4;
    if (memcmp(want, expanded, (size_t)C * 96) != 0) { fprintf(stderr, "expanded keys\n"); bad++; }
    for (c = 0; c < C; c++) {
        if (memcmp(pks + 32 * c, expanded + 96 * c + 64, 32) != 0) { fprintf(stderr, "pk %d\n", c); bad++; }
        if (memcmp(dids + AFC_DID_CHARS * c, "did:key:z7", 10) != 0) { fprintf(stderr, "did %d\n", c); bad++; }
    }
    if (strncmp((const char*)paths + AFC_DID_PATH_SLOT * 3, "m/44'/", 6) != 0) { fprintf(stderr, "path\n"); bad++; }
    for (i = 0; i < N; i++) {
        const char* b = (const char*)body + body_off[i];
        const size_t len = (size_t)(body_off[i + 1] - body_off[i]);
        if (len < 40 || strncmp(b, "{\"success\":true,\"identity_package\":{\"agent_did\":{\"did\":\"did:key:z", 62) != 0 || b[len - 1] != '}') {
            fprintf(stderr, "body %d\n", i); bad++;
        }
    }
    if (!contains(body, (size_t)body_off[N], "agent-two with 2 reasoners and 1 skills")) { fprintf(stderr, "message\n"); bad++; }
    /* argument errors */
    if (afc_did_register_batch(ctx, NULL, (const uint8_t*)server, strlen(server), nodes, node_off, agent_index, id_idx, ids, id_off, N, comp_off,
                               expanded, pks, dids, paths, flags, body, cap, body_off) != AFC_EINVAL) bad++;
    if (afc_did_register_batch(ctx, master, (const uint8_t*)server, strlen(server), nodes, node_off, agent_index, id_idx, ids, id_off, N, comp_off,
                               expanded, pks, dids, paths, flags, body, cap - 1, body_off) != AFC_EINVAL) bad++;
    memset(expanded, 0, sizeof expanded);
    free(body);
    afc_destroy(ctx);
    if (bad) { fprintf(stderr, "%d failed checks\n", bad); return 1; }
    printf("did_register ok\n");
    return 0;
}
