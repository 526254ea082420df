"""ORACLE — TEST INFRASTRUCTURE ONLY.  The reference's re-registration of a known agent restated on the CPU, independently of
agentfield_b200: RegisterAgent's branch for an agent the registry already holds (control-plane/internal/services/did_service.go:129-183),
PerformDifferentialAnalysis and setDifference (:757-847), buildExistingIdentityPackage (:940-986), handlePartialRegistration (:991-1045),
PartialRegisterAgent (:1049-1236) with generateReasonerPath / generateSkillPath (:870-937), and DeregisterComponents (:1239-1324).
Derivation, keys, JWKs and escaping come from oracle/ref_did.py (hashlib, `cryptography`, oracle.go_json), as for handleNewRegistration.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_did as RD  # noqa: E402

UNCHANGED, REMOVED, PARTIAL, INVALID = 0, 1, 2, 3            # AFC_DIDRR_*
GONE, NEW, KEPT = 1, 2, 1                                    # AFC_DIDRR_GONE, AFC_DIDRR_NEW, AFC_DID_KEPT


def stored_identity_json(ctype, did, public_key_jwk, path, function_name=b"") -> bytes:
    """buildExistingIdentityPackage's DIDIdentity (:940-986): PrivateKeyJWK "", PublicKeyJWK string(the stored json.RawMessage),
    FunctionName omitempty."""
    out = (b'{"did":' + RD._q(did) + b',"private_key_jwk":""' + b',"public_key_jwk":' + RD._q(public_key_jwk) + b',"derivation_path":' + RD._q(path) +
           b',"component_type":' + RD._q(ctype.encode()))
    if function_name:
        out += b',"function_name":' + RD._q(function_name)
    return out + b"}"


def reregister(master_seed: bytes, server_id: bytes, agent, reasoners, skills, agent_index: int):
    """RegisterAgent's branch for a known agent, one request.  agent: {"did", "public_key_jwk", "derivation_path", "reasoners", "skills"},
    the last two lists of (key, {"did", "public_key_jwk", "derivation_path", "function_name"}) in the registry's (any) order; reasoners,
    skills: the request's ids (bytes).  agent_index: the <a> of the new components' paths.  Returns {"state", "counts" (new reasoners, new
    skills, removed reasoners, removed skills), "body", "gone" (per registered component, in the given order), "id_flags" (per request
    id), "slots" (reasoners, skills: None or {"path", "seed", "pk", "did"})}.  A registered list that repeats a key is INVALID (no Go map
    holds one), with an empty body and no flags."""
    reg = (agent["reasoners"], agent["skills"])
    req = (reasoners, skills)
    nothing = {"state": INVALID, "counts": [0, 0, 0, 0], "body": b"", "gone": [[False] * len(reg[0]), [False] * len(reg[1])],
               "id_flags": [[0] * len(req[0]), [0] * len(req[1])], "slots": [None, None]}
    if any(len(set(k for k, _ in lst)) != len(lst) for lst in reg):
        return nothing
    h = RD.server_hash(server_id)
    maps = [dict(lst) for lst in reg]                              # existingAgent.Reasoners / .Skills
    new_ids, removed = [], []
    for kind in range(2):
        given = [x for x in req[kind] if x != b""]                 # extractReasonerIDs / extractSkillIDs
        existing = list(maps[kind])
        new_ids.append([x for x in given if x not in set(existing)])          # setDifference(new, existing): order and duplicates kept
        removed.append([x for x in existing if x not in set(given)])          # setDifference(existing, new)
    gone = [[k in set(removed[kind]) for k, _ in reg[kind]] for kind in range(2)]

    def package(agent_id, rmap, smap, msg):
        def map_json(m):
            return b"{" + b",".join(RD._q(k) + b":" + m[k] for k in sorted(m)) + b"}"
        return (b'{"success":true,"identity_package":{"agent_did":' + agent_id + b',"reasoner_dids":' + map_json(rmap) + b',"skill_dids":' +
                map_json(smap) + b',"agentfield_server_id":' + RD._q(server_id) + b'},"message":' + RD._q(msg) + b"}")
    agent_id = stored_identity_json("agent", agent["did"], agent["public_key_jwk"], agent["derivation_path"])

    def existing_maps():
        return [{k: stored_identity_json(t, v["did"], v["public_key_jwk"], v["derivation_path"], v["function_name"]) for k, v in maps[kind].items()}
                for kind, t in ((0, "reasoner"), (1, "skill"))]
    out = {"gone": gone, "id_flags": [[0] * len(req[0]), [0] * len(req[1])], "slots": [None, None]}
    if not (new_ids[0] or new_ids[1] or removed[0] or removed[1]):
        out.update(state=UNCHANGED, counts=[0, 0, 0, 0], body=package(agent_id, *existing_maps(), b"No changes detected, registration skipped"))
        return out
    for kind in range(2):                                          # DeregisterComponents
        for k in removed[kind]:
            del maps[kind][k]
    if not (new_ids[0] or new_ids[1]):
        msg = b"Registration updated: removed %d reasoners, %d skills" % (len(removed[0]), len(removed[1]))
        out.update(state=REMOVED, counts=[0, 0, len(removed[0]), len(removed[1])], body=package(agent_id, *existing_maps(), msg))
        return out
    new_maps = [{}, {}]                                            # PartialRegisterAgent
    for kind, ctype in ((0, "reasoner"), (1, "skill")):
        for ident in new_ids[kind]:
            path = RD.component_path(h, agent_index, kind, len(maps[kind]))     # len(existingAgent.Reasoners): not updated inside the loop
            c = RD._component(master_seed, path, ctype, ident)
            new_maps[kind][ident] = RD.identity_json(c)
            out["slots"][kind] = {"path": path, "seed": c["seed"], "pk": c["pk"], "did": c["did"]}
        lst = req[kind]
        for p, x in enumerate(lst):
            if x != b"" and x in set(new_ids[kind]):
                out["id_flags"][kind][p] = NEW | (KEPT if x not in lst[p + 1:] else 0)
    msg = b"Partial registration successful: %d new reasoners, %d new skills" % (len(new_maps[0]), len(new_maps[1]))
    out.update(state=PARTIAL, counts=[len(new_maps[0]), len(new_maps[1]), len(removed[0]), len(removed[1])],
               body=package(agent_id, new_maps[0], new_maps[1], msg))
    return out
