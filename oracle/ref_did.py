"""ORACLE — TEST INFRASTRUCTURE ONLY.  The reference's agent DID registration restated on the CPU, independently of agentfield_b200.

Follows control-plane/internal/services/did_service.go:186-365 (handleNewRegistration), :476-536 (generateDIDWithKeys,
derivePrivateKey, generateDIDKey), :538-575 (the JWK encoders), :578-582 (hashAgentFieldServerID), :653-723 (BackfillExistingNodes) and
pkg/types/did_types.go:106-121, 253-265 (field order).  Derivation with hashlib, public keys with `cryptography` (OpenSSL), strings
through oracle.go_json.escape_bytes; the JWK texts through Python's json module with sorted keys (json.Marshal of a map).
"""
import base64
import hashlib
import json

from cryptography.hazmat.primitives import serialization
from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey

from . import go_json as OJ


def fnv1a32(b: bytes) -> int:
    h = 0x811C9DC5
    for c in b:
        h = ((h ^ c) * 0x01000193) & 0xFFFFFFFF
    return h


def server_hash(server_id: bytes) -> int:
    """hashAgentFieldServerID: fnv.New32a, Sum32() % (1 << 31)."""
    return fnv1a32(server_id) % (1 << 31)


def agent_path(h, a):
    return b"m/44'/%d'/%d'" % (h, a)


def component_path(h, a, kind, j):
    """kind 0 = reasoner, 1 = skill."""
    return b"m/44'/%d'/%d'/%d'/%d'" % (h, a, kind, j)


def derive_seed(master_seed: bytes, path: bytes) -> bytes:
    return hashlib.sha256(master_seed + path).digest()


def public_key(seed: bytes) -> bytes:
    return Ed25519PrivateKey.from_private_bytes(seed).public_key().public_bytes(serialization.Encoding.Raw, serialization.PublicFormat.Raw)


def _b64(b: bytes) -> str:
    return base64.urlsafe_b64encode(b).rstrip(b"=").decode()


def did_key(pk: bytes) -> bytes:
    return b"did:key:z" + _b64(b"\xed\x01" + pk).encode()


def private_jwk(seed: bytes, pk: bytes) -> bytes:
    return json.dumps({"kty": "OKP", "crv": "Ed25519", "x": _b64(pk), "d": _b64(seed), "use": "sig", "alg": "EdDSA"}, sort_keys=True,
                      separators=(",", ":")).encode()


def public_jwk(pk: bytes) -> bytes:
    return json.dumps({"kty": "OKP", "crv": "Ed25519", "x": _b64(pk), "use": "sig", "alg": "EdDSA"}, sort_keys=True, separators=(",", ":")).encode()


def _q(s: bytes) -> bytes:
    return b'"' + OJ.escape_bytes(s) + b'"'


def identity_json(c) -> bytes:
    """json.Marshal(types.DIDIdentity) of one component."""
    out = (b'{"did":' + _q(c["did"]) + b',"private_key_jwk":' + _q(private_jwk(c["seed"], c["pk"])) + b',"public_key_jwk":' + _q(public_jwk(c["pk"])) +
           b',"derivation_path":' + _q(c["path"]) + b',"component_type":' + _q(c["type"].encode()))
    if c["type"] != "agent":
        out += b',"function_name":' + _q(c["id"])
    return out + b"}"


def _component(master_seed, path, ctype, ident=b""):
    seed = derive_seed(master_seed, path)
    pk = public_key(seed)
    return {"path": path, "seed": seed, "pk": pk, "did": did_key(pk), "type": ctype, "id": ident, "kept": True}


def register(master_seed: bytes, server_id: bytes, node_id: bytes, reasoners, skills, agent_index: int):
    """handleNewRegistration for one request (ids are bytes).  Returns {"components": [agent, non-empty reasoners in order, non-empty
    skills in order], each {"path", "seed", "pk", "did", "type", "id", "kept"}, "body": json.Marshal(DIDRegistrationResponse)}."""
    h = server_hash(server_id)
    comps = [_component(master_seed, agent_path(h, agent_index), "agent")]
    maps = []
    for kind, (ids, ctype) in enumerate(((reasoners, "reasoner"), (skills, "skill"))):
        m, j = {}, 0
        for ident in ids:
            if ident == b"":
                continue                                          # skipped: takes no index
            c = _component(master_seed, component_path(h, agent_index, kind, j), ctype, ident)
            if ident in m:
                m[ident]["kept"] = False                          # the map keeps the later assignment
            m[ident] = c
            comps.append(c)
            j += 1
        maps.append(m)

    def map_json(m):
        return b"{" + b",".join(_q(k) + b":" + identity_json(m[k]) for k in sorted(m)) + b"}"
    msg = b"Successfully registered agent %s with %d reasoners and %d skills" % (node_id, len(maps[0]), len(maps[1]))
    body = (b'{"success":true,"identity_package":{"agent_did":' + identity_json(comps[0]) + b',"reasoner_dids":' + map_json(maps[0]) +
            b',"skill_dids":' + map_json(maps[1]) + b',"agentfield_server_id":' + _q(server_id) + b'},"message":' + _q(msg) + b"}")
    return {"components": comps, "body": body}


def backfill_existing_nodes(master_seed: bytes, server_id: bytes, nodes, registered):
    """BackfillExistingNodes' loop: nodes is a list of (id, reasoner ids, skill ids); registered the set of node ids the registry holds
    (updated).  Each new node gets agent index len(registry) at its turn.  Returns [(node id, register(...))] for the new nodes."""
    out = []
    for node_id, reasoners, skills in nodes:
        if node_id in registered:
            continue
        out.append((node_id, register(master_seed, server_id, node_id, reasoners, skills, len(registered))))
        registered.add(node_id)
    return out
