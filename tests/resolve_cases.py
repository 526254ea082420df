"""Cases for DID resolution and DID documents (tests/resolve_oracle.py): the fixture's registry and requests, seeded random requests, the
directory a registry gives (each DID's first holder in registration order, as DIDService._identities takes it) and the golden file's
encoding."""
import hashlib
import json
import os

import numpy as np

import resolve_oracle as RO
from oracle import ref_did as RD

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "did_resolve_cases.json")
SEED = bytes(range(32))
SERVER_ID = b"af-server"


def _comp(path: bytes, fn: bytes, jwk=None):
    pk = RD.public_key(RD.derive_seed(SEED, path))
    return {"did": RD.did_key(pk), "derivation_path": path, "public_key_jwk": RD.public_jwk(pk) if jwk is None else jwk, "function_name": fn}


def _agent(a: int, reasoners, skills, jwk=None):
    h = RD.server_hash(SERVER_ID)
    ag = _comp(RD.agent_path(h, a), b"", jwk)
    del ag["function_name"]
    ag["reasoners"] = [(fn, _comp(RD.component_path(h, a, 0, j), fn)) for j, fn in enumerate(reasoners)]
    ag["skills"] = [(fn, _comp(RD.component_path(h, a, 1, j), fn)) for j, fn in enumerate(skills)]
    return ag


def fixture_registry():
    """Every kind, the root included; odd function names and paths; stored JWKs in many spellings; and duplicate DIDs from a
    re-registration after a removal: the re-registration gives each new component of a kind the same DID (DESIGN.md, K3)."""
    root_pk = RD.public_key(RD.derive_seed(SEED, RO.ROOT_PATH))
    agents = [_agent(0, [b"plan", b'q"uote\\back', b"<tag>&amp"], [b"search", b"line\xe2\x80\xa8sep", b"bad\xff\xfeutf8"]),
              _agent(1, [b"r1"], [b"s1"])]
    # re-registration of agent 1: r1 removed, r2 and r3 new, both at the slot's DID and path
    slot = _comp(RD.component_path(RD.server_hash(SERVER_ID), 1, 0, 1), b"")
    agents[1]["reasoners"] = [(fn, dict(slot, function_name=fn)) for fn in (b"r2", b"r3")]
    jwks = [b' { "kty" : "OKP" ,\n "crv":"Ed25519", "x":"abc", "use":"sig", "alg":"EdDSA" } ',        # whitespace
            b'{"x":"abc","kty":"OKP","alg":"EdDSA","use":"sig","crv":"Ed25519"}',                      # reordered keys
            b'{"n":1.50,"m":-0,"e":1E+2,"big":12345678901234567,"s":"a\\u003cb\\/c\\u00e9\\ud83d\\ude00","t":true,"f":false,"z":null}',
            b"null", b"[1,2]", b'"text"', b"{\"kty\":", b"", b'{"a":1,"a":2}', b'{"k\\u0061":1}', b'{"x":"\xff"}', b"  {}  ",
            b'{"pad":"' + b"x" * 4000 + b'"}', b'{"deep":' + b"[" * 40 + b"]" * 40 + b"}", b'{"tiny":1e-320}', b'{"huge":1e400}']
    for k, jwk in enumerate(jwks):
        agents.append(_agent(2 + k, [b"r"], [], jwk=jwk))
    agents.append(_agent(2 + len(jwks), [], [b"p" * 5000]))                                     # a resolve body over the cap
    odd = _agent(3 + len(jwks), [b"x"], [])
    odd["derivation_path"] = b"m/44'/\"<&>\\'/\xe2\x80\xa9/\xc0"
    agents.append(odd)
    return {"root_did": RD.did_key(root_pk), "root_pk": root_pk, "agents": agents}


def directory_entries(reg):
    """The directory a registry gives: each DID once, its first holder in registration order."""
    out = {}
    for e in RO.identities(reg):
        out.setdefault(e["did"], e)
    return list(out.values())


def fixture_requests(reg):
    reqs = [(RO.RESOLVE, b""), (RO.DOCUMENT, b""), (RO.RESOLVE, b"did:key:zUnknown"), (RO.DOCUMENT, b"did:key:zUnknown<&>\xff\xe2\x80\xa8"),
            (RO.DOCUMENT, b"x" * (1 << 20)), (RO.RESOLVE, b"\xc3\x28\xa0"), (RO.RESOLVE, reg["root_did"][:-1]), (RO.DOCUMENT, reg["root_did"][:20])]
    for e in directory_entries(reg):
        reqs += [(RO.RESOLVE, e["did"]), (RO.DOCUMENT, e["did"])]
    return reqs


def random_requests(reg, rng, n):
    """Half resolve, half document; mostly directory DIDs, some unknown, prefixes, empty and invalid UTF-8."""
    dids = [e["did"] for e in directory_entries(reg)]
    out = []
    for _ in range(n):
        kind = int(rng.integers(0, 2))
        r = rng.random()
        if r < 0.8:
            d = dids[int(rng.integers(0, len(dids)))]
        elif r < 0.85:
            d = dids[int(rng.integers(0, len(dids)))][:int(rng.integers(1, 40))]
        elif r < 0.9:
            d = b""
        else:
            d = bytes(rng.integers(0, 256, int(rng.integers(1, 80)), dtype=np.uint8))
        out.append((kind, d))
    return out


def _hex(x):
    return x.hex() if isinstance(x, bytes) else x


def _unhex(x):
    return bytes.fromhex(x)


def registry_to_json(reg):
    comp = lambda c: {k: v.hex() for k, v in c.items()}
    return {"root_did": reg["root_did"].hex(), "root_pk": reg["root_pk"].hex(),
            "agents": [dict({k: a[k].hex() for k in ("did", "derivation_path", "public_key_jwk")},
                            reasoners=[[fn.hex(), comp(c)] for fn, c in a["reasoners"]], skills=[[fn.hex(), comp(c)] for fn, c in a["skills"]])
                       for a in reg["agents"]]}


def registry_from_json(j):
    comp = lambda c: {k: bytes.fromhex(v) for k, v in c.items()}
    return {"root_did": _unhex(j["root_did"]), "root_pk": _unhex(j["root_pk"]),
            "agents": [dict({k: _unhex(a[k]) for k in ("did", "derivation_path", "public_key_jwk")},
                            reasoners=[(_unhex(fn), comp(c)) for fn, c in a["reasoners"]], skills=[(_unhex(fn), comp(c)) for fn, c in a["skills"]])
                       for a in j["agents"]]}


# In the golden file a request is [kind, hex, times] (the bytes repeated), and a body over 64 KB is stored as its SHA-256, so that the
# 1 MB request and its 404 document stay small.
BIG = 1 << 16


def request_json(kind, d):
    if len(d) > BIG and d == d[:1] * len(d):
        return [kind, d[:1].hex(), len(d)]
    return [kind, d.hex(), 1]


def outcomes_json(outs):
    enc = lambda b: None if b is None else {"sha256": hashlib.sha256(b).hexdigest()} if len(b) > BIG else b.hex()
    return [[st, enc(b), h] for st, b, h in outs]


def body_matches(stored, body) -> bool:
    if isinstance(stored, dict):
        return hashlib.sha256(body).hexdigest() == stored["sha256"]
    return stored is not None and _unhex(stored) == body


def load_fixture():
    """(registry, requests, expected): expected[i] the outcomes of request i as stored ((status, body as stored, host_ok))."""
    with open(FIXTURE) as f:
        fx = json.load(f)
    reg = registry_from_json(fx["registry"])
    reqs = [(k, _unhex(d) * t) for k, d, t in fx["requests"]]
    return reg, reqs, [[tuple(o) for o in outs] for outs in fx["expected"]]


def accepts_stored(outs, state, body) -> bool:
    """resolve_oracle.accepts over outcomes as the golden file stores them."""
    status = {0: 200, 1: 404, 2: 400}
    for st, b, host_ok in outs:
        if state == 3:
            if host_ok:
                return True
        elif status.get(state) == st and (st != 200 or len(body) <= RO.CAP) and body_matches(b, body):
            return True
    return False
