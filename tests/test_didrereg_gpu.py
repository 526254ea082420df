"""afc_did_reregister_batch[_dev] on the GPU against the oracle of tests/didrr_oracle.py (hashlib derivation, OpenSSL public keys): bodies,
states, counts, flags and key slots on 20 000 random known-agent requests; key slots against ctx.expand in both signing modes; the
host-buffer call against the _dev call (also with 97-request chunks and one request larger than a slot); a 1024-reasoner agent; no secret
left in staging memory; register -> re-register -> issue -> verify end to end; and DIDService.register_agents on a mixed batch."""
import hashlib
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import did_cases as DC
import didrr_cases as RC
import didrr_oracle as RR
from oracle import ref_did as RD

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def packed_call(keys, requests, master=RC.MASTER, server=RC.SERVER):
    A = RC.pack(requests)
    return keys.reregister_packed(master, server, A[0], A[1], A[2], *A[3:], append=False)


def dev_call(keys, requests, master=RC.MASTER, server=RC.SERVER):
    import torch
    A = RC.pack(requests)
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()  # noqa: E731
    R = keys.reregister_dev(t(np.frombuffer(master, dtype=np.uint8).copy(), np.uint8), server, t(A[0], np.uint8), t(A[1], np.int64),
                            t(A[2], np.int32), t(A[3], np.int64), t(A[4], np.uint8), t(A[5], np.int64), t(A[6], np.int64), t(A[7], np.uint8),
                            t(A[8], np.int64), len(requests), append=False)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in R.items()}
    out["counts"] = out["counts"].view(np.uint32)
    out["body_off"] = out["body_off"].view(np.uint64)
    return out


def compare(R, requests, want=None):
    want = want or RC.oracle(requests)
    body = R["body"].tobytes()
    g = k = 0
    for i, w in enumerate(want):
        assert body[int(R["body_off"][i]):int(R["body_off"][i + 1])] == w["body"], i
        assert R["state"][i] == w["state"] and list(R["counts"][i]) == w["counts"], i
        for kind in range(2):
            got = R["reg_flags"][g:g + len(w["gone"][kind])]
            assert [bool(x) for x in got] == w["gone"][kind], (i, kind)
            g += len(w["gone"][kind])
            assert list(R["id_flags"][k:k + len(w["id_flags"][kind])]) == w["id_flags"][kind], (i, kind)
            k += len(w["id_flags"][kind])
            s, t = w["slots"][kind], 2 * i + kind
            if s is None:
                assert not R["expanded"][t].any() and not R["pks"][t].any() and not R["dids"][t].any() and not R["paths"][t].any()
            else:
                assert R["pks"][t].tobytes() == s["pk"] and R["expanded"][t, 64:].tobytes() == s["pk"] and R["dids"][t].tobytes() == s["did"]
                assert R["paths"][t].tobytes().rstrip(b"\0") == s["path"]


@pytest.mark.parametrize("ct", [1, 0])
def test_key_slots_match_expand(ctx, ct):
    import agentfield_b200 as afb
    ctx.sign_configure(bool(ct))
    try:
        keys = afb.ExpandedKeys(ctx)
        reqs = RC.golden_requests()
        want = RC.oracle(reqs)
        for R in (packed_call(keys, reqs), dev_call(keys, reqs)):
            compare(R, reqs, want)
            live = [(2 * i + kind, s) for i, w in enumerate(want) for kind, s in enumerate(w["slots"]) if s]
            seeds = np.array([np.frombuffer(hashlib.sha256(RC.MASTER + s["path"]).digest(), dtype=np.uint8) for _, s in live])
            assert (R["expanded"][[t for t, _ in live]] == ctx.expand(seeds)).all()
    finally:
        ctx.sign_configure(True)


def test_random_20000(ctx):
    import agentfield_b200 as afb
    reqs = RC.random_requests(random.Random(41), 20000)
    R = dev_call(afb.ExpandedKeys(ctx), reqs)
    want = RC.oracle(reqs)
    assert {w["state"] for w in want} == {RR.UNCHANGED, RR.REMOVED, RR.PARTIAL, RR.INVALID}
    compare(R, reqs, want)


def test_host_call_equals_dev_call(ctx):
    import agentfield_b200 as afb
    keys = afb.ExpandedKeys(ctx)
    reqs = RC.random_requests(random.Random(43), 3000, max_reg=12)
    A, B = packed_call(keys, reqs), dev_call(keys, reqs)
    for k in A:
        assert (A[k] == B[k]).all(), k


CHUNK_SCRIPT = r"""
import random, sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import agentfield_b200 as afb, didrr_cases as RC
from test_didrereg_gpu import packed_call, dev_call, compare
ctx = afb.Context(0)
keys = afb.ExpandedKeys(ctx)
reqs = RC.random_requests(random.Random(47), 1000)
big = RC.random_requests(random.Random(48), 1, max_reg=0)[0]
jwk = b'{"x":"' + b"<" * 1200000 + b'"}'       # 16 stored JWKs of 1.2 MB: over 100 MB of body bound, past a slot's 96 MB
big["agent"]["reasoners"] = [(b"r%d" % k, {"did": b"d%d" % k, "public_key_jwk": jwk, "derivation_path": b"p", "function_name": b"f"}) for k in range(16)]
big["reasoners"] = [b"r%d" % k for k in range(1, 16)] + [b"added"]
reqs.insert(400, big)
A, B = packed_call(keys, reqs), dev_call(keys, reqs)
for k in A:
    assert (A[k] == B[k]).all(), k
compare(A, reqs)
print("chunks ok")
"""


def test_host_call_chunks_and_oversized_request():
    """97-request chunks (AFC_CHUNK_ITEMS is read once per process) and one request whose body bound is over 100 MB, which goes alone."""
    env = dict(os.environ, AFC_CHUNK_ITEMS="97", AFC_MIN_CHUNK_ITEMS="97")
    r = subprocess.run([sys.executable, "-c", CHUNK_SCRIPT, ROOT], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "chunks ok" in r.stdout, r.stderr[-3000:]


def test_agent_with_1024_reasoners(ctx):
    import agentfield_b200 as afb
    agent = RC.registered(RC.MASTER, RC.SERVER, b"wide", [b"reasoner_%d" % k for k in range(1024)], [b"s"], 5)
    keep = [b"reasoner_%d" % k for k in range(1024) if k % 7]
    reqs = [{"agent_node_id": b"wide", "agent": agent, "reasoners": keep + [b"added_%d" % k for k in range(100)], "skills": [b"s"], "agent_index": 5},
            {"agent_node_id": b"wide", "agent": agent, "reasoners": [b"reasoner_%d" % k for k in range(1024)], "skills": [b"s"], "agent_index": 5},
            {"agent_node_id": b"wide", "agent": agent, "reasoners": keep, "skills": [], "agent_index": 5}]
    R = dev_call(afb.ExpandedKeys(ctx), reqs)
    compare(R, reqs)
    assert list(R["state"]) == [RR.PARTIAL, RR.UNCHANGED, RR.REMOVED]


def test_host_call_leaves_no_secret_in_staging(ctx):
    """After the host-buffer call, the context's staging memory holds neither the master seed nor any derived seed, expanded-key half or
    private JWK "d"; a public id it staged is still there, which shows the search sees that memory."""
    import base64
    import ctypes as C
    import agentfield_b200 as afb
    from agentfield_b200 import _abi
    lib = _abi.load()
    master = bytes(range(0xC0, 0xE0))
    reqs = RC.random_requests(random.Random(53), 500, mix=(0.1, 0.1, 0.8))
    for i, r in enumerate(reqs):
        r["reasoners"] = list(r["reasoners"]) + [b"staged-id-%06d" % i]
    R = packed_call(afb.ExpandedKeys(ctx), reqs, master=master)
    want = RC.oracle(reqs, master=master)

    def hits(pattern):
        h = C.c_uint64()
        _abi.check(lib.afc_staging_find(ctx.handle, pattern, len(pattern), C.byref(h)), ctx.handle)
        return h.value
    assert hits(b"staged-id-000123") > 0
    assert hits(master) == 0
    slots = [s for w in want for s in w["slots"] if s]
    assert len(slots) > 400
    for s in slots[::23]:
        assert hits(s["seed"]) == 0
        assert hits(base64.urlsafe_b64encode(s["seed"]).rstrip(b"=")) == 0
    for t in range(0, 2 * len(reqs), 37):
        if R["expanded"][t].any():
            assert hits(R["expanded"][t, :32].tobytes()) == 0 and hits(R["expanded"][t, 32:64].tobytes()) == 0


def test_register_reregister_issue_verify(ctx):
    import agentfield_b200 as afb
    from agentfield_b200 import _abi, services
    keys = afb.ExpandedKeys(ctx)
    svc = services.DIDService(keys, DC.MASTER, DC.SERVER)
    svc.register_agents_batch([{"agent_node_id": "n1", "reasoners": ["a", "b", "c"], "skills": ["s"]},
                               {"agent_node_id": "n2", "reasoners": [], "skills": ["t"]}])
    res = svc.reregister_agents_batch([{"agent_node_id": "n1", "reasoners": ["a", "c", "d", "d"], "skills": []},
                                       {"agent_node_id": "n2", "reasoners": ["x"], "skills": ["t", "u"]}])
    assert [r["state"] for r in res] == [_abi.DIDRR_PARTIAL, _abi.DIDRR_PARTIAL]
    n1, n2 = svc.agent_nodes[b"n1"], svc.agent_nodes[b"n2"]
    assert set(n1["reasoners"]) == {b"a", b"c", b"d"} and set(n1["skills"]) == set()
    assert set(n2["reasoners"]) == {b"x"} and set(n2["skills"]) == {b"t", b"u"}
    new_dids = [n1["reasoners"][b"d"]["did"], n2["reasoners"][b"x"]["did"], n2["skills"][b"u"]["did"]]
    assert new_dids[0] == res[0]["slots"][0]["did"]
    ks = afb.KeySet([keys.public_key(d) for d in new_dids], ctx, dids=new_dids)
    reqs = [{"vc_id": "vc-%d" % k, "caller_did": d, "issuance_date": "2026-10-16T00:00:00Z", "execution_id": "e%d" % k, "workflow_id": "w",
             "session_id": "s", "caller_type": "agent", "agent_node_did": d, "target_did": "", "function_name": "f",
             "timestamp": "2026-10-16T00:00:00Z", "status": "succeeded", "error_message": "", "proof_created": "2026-10-16T00:00:00Z",
             "duration_ms": 5, "input": b"{}", "output": b"[1]"} for k, d in enumerate(new_dids)]
    issued = keys.issue(reqs)
    st, _ = ks.verify_stored(_abi.DOC_EXECUTION_VC, [r["vc_document"] for r in issued])
    assert (st == _abi.VC_VALID).all()
    again = svc.reregister_agents_batch([{"agent_node_id": "n1", "reasoners": ["a", "c", "d"], "skills": []}])
    assert again[0]["state"] == _abi.DIDRR_UNCHANGED
    with pytest.raises(ValueError):
        svc.reregister_agents_batch([{"agent_node_id": "unknown", "reasoners": [], "skills": []}])
    with pytest.raises(ValueError):
        svc.reregister_agents_batch([{"agent_node_id": "n1", "reasoners": [], "skills": []}] * 2)


def test_register_agents_mixed_batch_equals_oracle_in_order(ctx):
    import agentfield_b200 as afb
    from agentfield_b200 import services
    rng = random.Random(59)
    svc = services.DIDService(afb.ExpandedKeys(ctx), DC.MASTER, DC.SERVER)
    reg = {}                                                      # the oracle's registry: node -> agent record (RR.reregister's form)

    def oracle_apply(r):
        node = r["agent_node_id"]
        if node not in reg:
            a = RC.registered(DC.MASTER, DC.SERVER, node, r["reasoners"], r["skills"], len(reg))
            reg[node] = a
            return RD.register(DC.MASTER, DC.SERVER, node, r["reasoners"], r["skills"], len(reg) - 1)["body"]
        a = reg[node]
        w = RR.reregister(DC.MASTER, DC.SERVER, a, r["reasoners"], r["skills"], int(a["derivation_path"].split(b"/")[3][:-1]))
        for kind, name in ((0, "reasoners"), (1, "skills")):
            m = dict(a[name])
            for (key, _), gone in zip(a[name], w["gone"][kind]):
                if gone:
                    del m[key]
            s = w["slots"][kind]
            for x, f in zip(r[name], w["id_flags"][kind]):
                if f == RR.NEW | RR.KEPT:
                    m[x] = {"did": s["did"], "public_key_jwk": RD.public_jwk(s["pk"]), "derivation_path": s["path"], "function_name": x}
            a[name] = list(m.items())
        return w["body"]
    pool = [b"r%d" % k for k in range(8)]
    for rnd in range(4):
        batch = []
        for k in rng.sample(range(60), 40):
            batch.append({"agent_node_id": b"node-%d" % k, "reasoners": rng.sample(pool, rng.randrange(5)) + ([b""] if rng.random() < 0.2 else []),
                          "skills": rng.sample(pool, rng.randrange(3))})
        got = svc.register_agents(batch)
        want = [oracle_apply(r) for r in batch]
        assert [g["body"] for g in got] == want, rnd
    with pytest.raises(ValueError):
        svc.register_agents([{"agent_node_id": b"node-1", "reasoners": [], "skills": []}] * 2)
