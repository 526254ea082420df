"""Known-agent re-registration cases shared by the CPU and GPU tests and the fixture generator: requests as afc_did_reregister_batch
packs them, and what the oracle (tests/didrr_oracle.py) says the reference returns for them.

A request is {"agent_node_id", "agent": {"did", "public_key_jwk", "derivation_path", "reasoners", "skills"}, "reasoners", "skills",
"agent_index"}; the agent's lists hold (key, {"did", "public_key_jwk", "derivation_path", "function_name"}) pairs."""
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_did as RD  # noqa: E402
import did_cases as DC  # noqa: E402
import didrr_oracle as RR  # noqa: E402

MASTER, SERVER, ESCAPES = DC.MASTER, DC.SERVER, DC.ESCAPES
COLS = ("did", "public_key_jwk", "derivation_path", "function_name")


def _cat(xs):
    off = np.zeros(len(xs) + 1, dtype=np.uint64)
    if xs:
        off[1:] = np.cumsum([len(x) for x in xs])
    return np.frombuffer(b"".join(xs) + b"\0", dtype=np.uint8).copy(), off


def pack(requests):
    """-> (agent_cols, agent_col_off, agent_index, id_idx, ids, id_off, reg_idx, reg_cols, reg_col_off) as uint8 / uint32 / uint64 arrays."""
    acols, flat, idx, rflat, ridx = [], [], [0], [], [0]
    for r in requests:
        a = r["agent"]
        acols += [a["did"], a["public_key_jwk"], a["derivation_path"]]
        for kind in ("reasoners", "skills"):
            flat += list(r[kind])
            idx.append(len(flat))
            for key, c in a[kind]:
                rflat += [key] + [c[k] for k in COLS]
            ridx.append(len(rflat) // 5)
    agent_cols, agent_col_off = _cat(acols)
    ids, id_off = _cat(flat)
    reg_cols, reg_col_off = _cat(rflat)
    ai = np.array([r["agent_index"] for r in requests], dtype=np.uint64).astype(np.uint32)
    return (agent_cols, agent_col_off, ai, np.array(idx, dtype=np.uint64), ids, id_off, np.array(ridx, dtype=np.uint64), reg_cols, reg_col_off)


def oracle(requests, master=MASTER, server=SERVER):
    return [RR.reregister(master, server, r["agent"], r["reasoners"], r["skills"], r["agent_index"]) for r in requests]


def registered(master, server, node_id, reasoners, skills, agent_index):
    """A known agent as handleNewRegistration leaves it in the registry (the canonical JWK spelling, function_name = the id)."""
    w = RD.register(master, server, node_id, reasoners, skills, agent_index)
    comps = w["components"]
    agent = {"did": comps[0]["did"], "public_key_jwk": RD.public_jwk(comps[0]["pk"]), "derivation_path": comps[0]["path"], "reasoners": [],
             "skills": []}
    for kind, t in (("reasoners", "reasoner"), ("skills", "skill")):
        m = {}
        for c in comps[1:]:
            if c["type"] == t and c["kept"]:
                m[c["id"]] = {"did": c["did"], "public_key_jwk": RD.public_jwk(c["pk"]), "derivation_path": c["path"], "function_name": c["id"]}
        agent[kind] = list(m.items())
    return agent


def _fake_component(rng, key, kind):
    """A stored component whose columns need not come from a key: the call copies them as stored."""
    did = b"did:key:z" + bytes(rng.choice(b"ABCDEFabcdef0123456789-_") for _ in range(46))
    u = rng.random()
    if u < 0.1:
        jwk = b'{ "kty": "OKP", "crv": "Ed25519", "x": "%s" }' % did[9:52]             # a non-canonical spelling, kept as stored
    elif u < 0.15:
        jwk = rng.choice(ESCAPES) + b"\n<jwk>"
    else:
        jwk = b'{"alg":"EdDSA","crv":"Ed25519","kty":"OKP","use":"sig","x":"%s"}' % did[9:52]
    path = b"m/44'/%d'/%d'/%d'/%d'" % (rng.randrange(2 ** 31), rng.randrange(1000), kind, rng.randrange(64))
    fn = b"" if rng.random() < 0.1 else (rng.choice(ESCAPES) if rng.random() < 0.05 else key)
    return {"did": did, "public_key_jwk": jwk, "derivation_path": path, "function_name": fn}


def random_requests(rng: random.Random, n, max_reg=8, max_new=4, esc=0.05, invalid=0.01, mix=(0.4, 0.3, 0.3)):
    """Known agents with 0..max_reg registered reasoners and skills, and requests that keep them (in any order, with repeats and empty
    ids), drop some, and add new ids drawn from a small pool (so repeats are common).  mix: the fractions of unchanged, removals-only and
    partial requests (before escapes and repeats shift them)."""
    pool = [b"fn_%d" % k for k in range(6)] + [b"new_%d" % k for k in range(4)]
    out = []
    for i in range(n):
        agent = {"did": b"did:key:zAgent%d" % i, "public_key_jwk": b'{"kty":"OKP","x":"a%d"}' % i,
                 "derivation_path": b"m/44'/%d'/%d'" % (rng.randrange(2 ** 31), i), "reasoners": [], "skills": []}
        req = {}
        u = rng.random()
        mode = 0 if u < mix[0] else 1 if u < mix[0] + mix[1] else 2
        for kind, name in ((0, "reasoners"), (1, "skills")):
            keys = []
            for _ in range(rng.randrange(max_reg + 1)):
                k = rng.choice(ESCAPES) if rng.random() < esc else rng.choice(pool) if rng.random() < 0.5 else b"comp_%d" % rng.randrange(10 ** 6)
                if k not in keys:
                    keys.append(k)
            if keys and rng.random() < invalid:
                keys.append(keys[0])
            agent[name] = [(k, _fake_component(rng, k, kind)) for k in keys]
            ids = list(keys)
            if mode >= 1 and ids and rng.random() < 0.6:
                del ids[rng.randrange(len(ids))]
            if mode == 2 and rng.random() < 0.7:
                ids += [rng.choice(pool + ESCAPES) + (b"" if rng.random() < 0.7 else b"!") for _ in range(rng.randrange(1, max_new + 1))]
            ids = [x for x in ids if x is not None]
            rng.shuffle(ids)
            if ids and rng.random() < 0.2:
                ids.append(rng.choice(ids))
            if rng.random() < 0.1:
                ids.insert(rng.randrange(len(ids) + 1), b"")
            req[name] = ids
        out.append({"agent_node_id": b"node-%d" % i, "agent": agent, "reasoners": req["reasoners"], "skills": req["skills"],
                    "agent_index": rng.randrange(2 ** 32) if rng.random() < 0.1 else i})
    return out


def golden_requests():
    """The fixture's requests: every state; repeated new ids; the shared path index, also a new reasoner that gets a surviving
    component's DID after a removal; empty ids and lists; ids and columns that need escaping; a stored JWK in a non-canonical spelling;
    an empty stored function_name."""
    reg = lambda node, rs, ss, a: registered(MASTER, SERVER, node, rs, ss, a)  # noqa: E731
    out = []

    def add(node, agent, rs, ss, a):
        out.append({"agent_node_id": node, "agent": agent, "reasoners": rs, "skills": ss, "agent_index": a})
    base = reg(b"same", [b"r0", b"r1", b"r2"], [b"s0"], 3)
    add(b"same", base, [b"r2", b"r0", b"r1", b"r0", b""], [b"s0"], 3)                                     # unchanged, any order
    add(b"bare", reg(b"bare", [], [], 4), [], [], 4)                                                     # unchanged, empty lists
    add(b"removed", reg(b"removed", [b"a", b"b", b"c"], [b"x", b"y"], 5), [b"a", b"c"], [b""], 5)        # removals only
    add(b"partial", reg(b"partial", [b"a"], [], 6), [b"a", b"n2", b"n1", b"n2", b""], [b"t1", b"t1"], 6)  # repeated new ids, shared key
    # r0 removed: len(Reasoners) = 2 = r2's index, so the new reasoner gets r2's path and DID
    add(b"collide", reg(b"collide", [b"r0", b"r1", b"r2"], [], 7), [b"r1", b"r2", b"fresh"], [], 7)
    add(b"swap", reg(b"swap", [b"old"], [b"s"], 8), [b"new"], [], 8)                                     # removals and additions
    esc = reg(b"esc", ESCAPES[:4], ESCAPES[4:6], 9)
    add(b"esc", esc, ESCAPES[:3] + [ESCAPES[7]], ESCAPES[4:6] + [ESCAPES[10]], 9)
    odd = reg(b"odd", [b"k1", b"k2"], [b"s1"], 10)
    odd["public_key_jwk"] = b'{ "kty" : "OKP",\n  "crv": "Ed25519", "x": "<\xe2\x80\xa8\xff&>" }'        # stored as the client sent it
    odd["reasoners"][0][1]["public_key_jwk"] = b'{"x":"\x01\x1f","kty":"OKP"}'
    odd["reasoners"][1][1]["function_name"] = b""                                                      # omitted
    odd["did"] = b"did:key:z<odd>\xe2\x80\xa9"
    add(b"odd", odd, [b"k1", b"k2"], [b"s1"], 10)
    add(b"odd-removed", odd, [b"k2"], [], 10)
    add(b"invalid", {**reg(b"invalid", [b"a"], [], 11), "reasoners": [(b"a", {"did": b"d1", "public_key_jwk": b"{}", "derivation_path": b"p",
                                                                             "function_name": b"a"})] * 2}, [b"a", b"b"], [], 11)
    add(b"big-index", reg(b"big-index", [b"q"], [b"s"], 2 ** 32 - 1), [b"q", b"w"], [b"z"], 2 ** 32 - 1)
    return out


def to_json(r):
    """A request with its byte strings as hex (the fixture's form)."""
    comp = lambda lst: [[k.hex(), {c: v[c].hex() for c in COLS}] for k, v in lst]  # noqa: E731
    a = r["agent"]
    return {"agent_node_id": r["agent_node_id"].hex(), "agent_index": r["agent_index"], "reasoners": [x.hex() for x in r["reasoners"]],
            "skills": [x.hex() for x in r["skills"]],
            "agent": {"did": a["did"].hex(), "public_key_jwk": a["public_key_jwk"].hex(), "derivation_path": a["derivation_path"].hex(),
                      "reasoners": comp(a["reasoners"]), "skills": comp(a["skills"])}}


def from_json(j):
    comp = lambda lst: [(bytes.fromhex(k), {c: bytes.fromhex(v[c]) for c in COLS}) for k, v in lst]  # noqa: E731
    a = j["agent"]
    return {"agent_node_id": bytes.fromhex(j["agent_node_id"]), "agent_index": j["agent_index"], "reasoners": [bytes.fromhex(x) for x in j["reasoners"]],
            "skills": [bytes.fromhex(x) for x in j["skills"]],
            "agent": {"did": bytes.fromhex(a["did"]), "public_key_jwk": bytes.fromhex(a["public_key_jwk"]),
                      "derivation_path": bytes.fromhex(a["derivation_path"]), "reasoners": comp(a["reasoners"]), "skills": comp(a["skills"])}}
