"""afc_did_register_batch[_dev] on the GPU against oracle/ref_did.py (hashlib derivation, OpenSSL public keys): keys in both signing modes,
bodies on 20 000 random registrations, the host-buffer call against the _dev call (also with 97-request chunks and one request larger
than a slot), register -> issue -> verify end to end, argument errors, empty batches, 2^20 components, and DIDService's backfill."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import did_cases as DC
from oracle import ref_did as RD

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def packed_call(keys, requests, agent_base=0, server=DC.SERVER, master=DC.MASTER):
    nodes, node_off, id_idx, ids, id_off = DC.pack(requests)
    ai = np.arange(agent_base, agent_base + len(requests), dtype=np.uint64).astype(np.uint32)
    return keys.register_packed(master, server, nodes, node_off, ai, id_idx, ids, id_off, append=False)


def dev_call(keys, requests, agent_base=0, server=DC.SERVER, master=DC.MASTER):
    import torch
    nodes, node_off, id_idx, ids, id_off = DC.pack(requests)
    ai = np.arange(agent_base, agent_base + len(requests), dtype=np.uint64).astype(np.uint32)
    t = lambda a, dt: torch.from_numpy(a.view(dt)).cuda()  # noqa: E731
    R = keys.register_dev(t(np.frombuffer(master, dtype=np.uint8).copy(), np.uint8), server, t(nodes, np.uint8), t(node_off, np.int64),
                          t(ai, np.int32), t(id_idx, np.int64), t(ids, np.uint8), t(id_off, np.int64), len(requests), append=False)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in R.items()}


def compare(R, requests, agent_base=0, check_seeds=None):
    want = DC.oracle(requests, agent_base)
    body = R["body"].tobytes()
    for i, w in enumerate(want):
        assert body[int(R["body_off"][i]):int(R["body_off"][i + 1])] == w["body"], i
        c0 = int(R["comp_off"][i])
        assert int(R["comp_off"][i + 1]) - c0 == len(w["components"])
        for k, wc in enumerate(w["components"]):
            c = c0 + k
            assert R["pks"][c].tobytes() == wc["pk"] and R["expanded"][c, 64:].tobytes() == wc["pk"]
            assert R["dids"][c].tobytes() == wc["did"]
            assert R["paths"][c].tobytes().rstrip(b"\0") == wc["path"]
            assert bool(R["flags"][c]) == wc["kept"]


@pytest.mark.parametrize("ct", [1, 0])
def test_keys_match_openssl_and_expand(ctx, ct):
    import agentfield_b200 as afb
    ctx.sign_configure(bool(ct))
    try:
        keys = afb.ExpandedKeys(ctx)
        reqs = DC.golden_requests()
        for R in (packed_call(keys, reqs, 7), dev_call(keys, reqs, 7)):
            compare(R, reqs, 7)
            seeds = np.array([np.frombuffer(c["seed"], dtype=np.uint8) for w in DC.oracle(reqs, 7) for c in w["components"]])
            assert (R["expanded"] == ctx.expand(seeds)).all()
    finally:
        ctx.sign_configure(True)


def test_bodies_random_20000(ctx):
    import agentfield_b200 as afb
    keys = afb.ExpandedKeys(ctx)
    reqs = DC.random_requests(random.Random(5), 20000, max_ids=6)
    R = dev_call(keys, reqs, 1000)
    compare(R, reqs, 1000)


def test_host_call_equals_dev_call(ctx):
    import agentfield_b200 as afb
    keys = afb.ExpandedKeys(ctx)
    reqs = DC.random_requests(random.Random(9), 3000, max_ids=12)
    A, B = packed_call(keys, reqs, 3), dev_call(keys, reqs, 3)
    for k in A:
        assert (A[k] == B[k]).all(), k


CHUNK_SCRIPT = r"""
import random, sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import agentfield_b200 as afb, did_cases as DC
from test_didreg_gpu import packed_call, dev_call
ctx = afb.Context(0)
keys = afb.ExpandedKeys(ctx)
reqs = DC.random_requests(random.Random(13), 1000, max_ids=8)
big = {"agent_node_id": b"big", "reasoners": [b"r%d_%s" % (k, b"x" * 200) for k in range(500000)], "skills": [b"s"]}
reqs.insert(400, big)
A, B = packed_call(keys, reqs, 0), dev_call(keys, reqs, 0)
for k in A:
    assert (A[k] == B[k]).all(), k
print("chunks ok")
"""


def test_host_call_chunks_and_oversized_request():
    """97-request chunks (AFC_CHUNK_ITEMS is read once per process) and one request of 500 000 ids (over 100 MB staged: a slot's budget
    is 96 MB) that goes alone."""
    env = dict(os.environ, AFC_CHUNK_ITEMS="97", AFC_MIN_CHUNK_ITEMS="97")
    r = subprocess.run([sys.executable, "-c", CHUNK_SCRIPT, ROOT], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "chunks ok" in r.stdout, r.stderr[-3000:]


def test_register_issue_verify(ctx):
    import agentfield_b200 as afb
    from agentfield_b200 import _abi, services
    keys = afb.ExpandedKeys(ctx)
    svc = services.DIDService(keys, DC.MASTER, DC.SERVER)
    res = svc.register_agents_batch(DC.golden_requests())
    comps = [c for r in res for c in r["components"]]
    ks = afb.KeySet([c["pk"] for c in comps], ctx, dids=[c["did"] for c in comps])
    reqs = []
    for k, c in enumerate(comps):
        reqs.append({"vc_id": "vc-%d" % k, "caller_did": c["did"], "issuance_date": "2026-10-16T00:00:00Z", "execution_id": "e%d" % k,
                     "workflow_id": "w", "session_id": "s", "caller_type": "agent", "agent_node_did": c["did"], "target_did": "",
                     "function_name": "f", "timestamp": "2026-10-16T00:00:00Z", "status": "succeeded", "error_message": "",
                     "proof_created": "2026-10-16T00:00:00Z", "duration_ms": 5, "input": b"{}", "output": b"[1]"})
    issued = keys.issue(reqs)
    st, _ = ks.verify_stored(_abi.DOC_EXECUTION_VC, [r["vc_document"] for r in issued])
    assert (st == _abi.VC_VALID).all()
    with pytest.raises(ValueError):
        svc.register_agents_batch([{"agent_node_id": "bare-agent", "reasoners": [], "skills": []}])
    with pytest.raises(ValueError):
        svc.register_agents_batch([{"agent_node_id": "x", "reasoners": [], "skills": []}] * 2)


def test_argument_errors_and_empty(ctx):
    import agentfield_b200 as afb
    from agentfield_b200 import _abi
    lib = _abi.load()
    keys = afb.ExpandedKeys(ctx)
    reqs = DC.golden_requests()[:3]
    nodes, node_off, id_idx, ids, id_off = DC.pack(reqs)
    n, m = len(reqs), int(id_idx[-1])
    ai = np.zeros(n, dtype=np.uint32)
    ms = np.frombuffer(DC.MASTER, dtype=np.uint8).copy()
    cap = lib.afc_did_register_bound(_abi.ptr(node_off), _abi.ptr(id_idx), _abi.ptr(id_off), n, len(DC.SERVER))
    out = [np.zeros(n + 1, dtype=np.uint64), np.zeros((n + m) * 96, dtype=np.uint8), np.zeros((n + m) * 32, dtype=np.uint8),
           np.zeros((n + m) * 55, dtype=np.uint8), np.zeros((n + m) * 48, dtype=np.uint8), np.zeros(n + m, dtype=np.uint8), np.zeros(cap, dtype=np.uint8)]
    boff = np.zeros(n + 1, dtype=np.uint64)

    def call(ms=ms, node_off=node_off, id_idx=id_idx, id_off=id_off, cap=cap, n=n, body=out[6]):
        return lib.afc_did_register_batch(ctx.handle, _abi.ptr(ms), DC.SERVER, len(DC.SERVER), _abi.ptr(nodes), _abi.ptr(node_off), _abi.ptr(ai),
                                          _abi.ptr(id_idx), _abi.ptr(ids), _abi.ptr(id_off), n, *[_abi.ptr(x) for x in out[:6]], _abi.ptr(body), cap,
                                          _abi.ptr(boff))
    assert call() == _abi.AFC_OK
    assert call(ms=None) == _abi.AFC_EINVAL
    assert call(body=None) == _abi.AFC_EINVAL
    assert call(cap=cap - 1) == _abi.AFC_EINVAL
    back = id_idx.copy(); back[2] = back[1] - 1 if back[1] else 5
    assert call(id_idx=back) == _abi.AFC_EINVAL
    bo = id_off.copy(); bo[1], bo[2] = bo[2], bo[1]
    assert bo[1] > bo[2] and call(id_off=bo) == _abi.AFC_EINVAL
    no = node_off.copy(); no[1] = no[2] + 1
    assert call(node_off=no) == _abi.AFC_EINVAL
    boff[:] = 7; out[0][:] = 7
    assert call(n=0, cap=0) == _abi.AFC_OK and boff[0] == 0 and out[0][0] == 0
    assert packed_call(keys, [])["comp_off"].tolist() == [0]
    empty = [{"agent_node_id": b"e%d" % k, "reasoners": [b""] * 3, "skills": [b""]} for k in range(5)]
    for R in (packed_call(keys, empty), dev_call(keys, empty)):
        compare(R, empty)
        assert R["comp_off"].tolist() == list(range(6))


def test_two_to_the_twenty_components(ctx):
    import agentfield_b200 as afb
    keys = afb.ExpandedKeys(ctx)
    rng = random.Random(17)
    reqs = [{"agent_node_id": b"agent-%d" % i, "reasoners": [b"summarize_text_%d" % rng.randrange(10 ** 6) for _ in range(31)],
             "skills": [b"skill_%d" % k for k in range(32)]} for i in range(16384)]
    R = dev_call(keys, reqs)
    assert int(R["comp_off"][-1]) == 2 ** 20
    body = R["body"].tobytes()
    for i in range(0, 16384, 997):
        w = DC.oracle([reqs[i]], i)[0]
        assert body[int(R["body_off"][i]):int(R["body_off"][i + 1])] == w["body"]
        c0 = int(R["comp_off"][i])
        assert [R["pks"][c0 + k].tobytes() for k in range(64)] == [c["pk"] for c in w["components"]]


def test_backfill_equals_sequential_loop(ctx):
    import agentfield_b200 as afb
    from agentfield_b200 import services
    rng = random.Random(23)
    nodes = DC.random_requests(rng, 200, max_ids=5)
    for k in range(0, 200, 10):
        nodes[k]["agent_node_id"] = b"node-%d" % (k // 2)         # some repeat an earlier node
    svc = services.DIDService(afb.ExpandedKeys(ctx), DC.MASTER, DC.SERVER)
    first = svc.register_agents_batch(nodes[:3])
    got = svc.backfill_existing_nodes(nodes)
    registered = set(r["agent_node_id"] for r in nodes[:3])
    want = RD.backfill_existing_nodes(DC.MASTER, DC.SERVER, [(r["agent_node_id"], r["reasoners"], r["skills"]) for r in nodes], registered)
    assert len(first) == 3 and [g["body"] for g in got] == [w["body"] for _, w in want]
    assert len(svc.agent_nodes) == len(registered)


def test_dev_argument_errors(ctx):
    import torch
    from agentfield_b200 import _abi
    lib = _abi.load()
    reqs = DC.golden_requests()[:3]
    nodes, node_off, id_idx, ids, id_off = DC.pack(reqs)
    n, m = len(reqs), int(id_idx[-1])
    cap = lib.afc_did_register_bound(_abi.ptr(node_off), _abi.ptr(id_idx), _abi.ptr(id_off), n, len(DC.SERVER))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    d = {"ms": t(np.frombuffer(DC.MASTER, dtype=np.uint8).copy()), "nodes": t(nodes), "node_off": t(node_off.view(np.int64)),
         "ai": t(np.zeros(n, dtype=np.int32)), "id_idx": t(id_idx.view(np.int64)), "ids": t(ids), "id_off": t(id_off.view(np.int64)),
         "comp_off": torch.zeros(n + 1, dtype=torch.int64, device="cuda"), "exp": torch.zeros((n + m + 1) * 96, dtype=torch.uint8, device="cuda"),
         "pks": torch.zeros((n + m) * 32, dtype=torch.uint8, device="cuda"), "dids": torch.zeros((n + m) * 55, dtype=torch.uint8, device="cuda"),
         "paths": torch.zeros((n + m) * 48, dtype=torch.uint8, device="cuda"), "flags": torch.zeros(n + m, dtype=torch.uint8, device="cuda"),
         "body": torch.zeros(cap, dtype=torch.uint8, device="cuda"), "body_off": torch.zeros(n + 1, dtype=torch.int64, device="cuda")}

    def call(cap=cap, **kw):
        a = dict(d, **kw)
        p = lambda k: a[k] if isinstance(a[k], int) or a[k] is None else _abi.ptr(a[k])  # noqa: E731
        rc = lib.afc_did_register_batch_dev(ctx.handle, p("ms"), DC.SERVER, len(DC.SERVER), p("nodes"), p("node_off"), p("ai"), p("id_idx"), p("ids"),
                                            p("id_off"), n, p("comp_off"), p("exp"), p("pks"), p("dids"), p("paths"), p("flags"), p("body"), cap,
                                            p("body_off"), None)
        torch.cuda.synchronize()
        return rc
    assert call() == _abi.AFC_OK
    assert int(d["body_off"][n]) == sum(len(w["body"]) for w in DC.oracle(reqs))
    for k in ("ms", "nodes", "node_off", "ai", "id_idx", "id_off", "comp_off", "exp", "pks", "dids", "paths", "flags", "body", "body_off"):
        assert call(**{k: None}) == _abi.AFC_EINVAL, k
    assert call(cap=cap - 1) == _abi.AFC_EINVAL
    assert call(exp=_abi.ptr(d["exp"]) + 8) == _abi.AFC_EINVAL                 # expanded keys not 16-byte aligned
    back = id_idx.copy(); back[0], back[2 * n] = back[2 * n], back[0]
    assert call(id_idx=t(back.view(np.int64))) == _abi.AFC_EINVAL               # the id range runs backwards
    nb = node_off.copy(); nb[0], nb[n] = nb[n], nb[0]
    assert call(node_off=t(nb.view(np.int64))) == _abi.AFC_EINVAL


def test_host_call_leaves_no_secret_in_staging(ctx):
    """After the host-buffer call, the context's staging memory (every lane's device slots and pinned bounce buffers) holds neither the
    master seed nor any derived seed, expanded key or private JWK text; the public node ids it staged are still there, which shows the
    search sees that memory."""
    import base64
    import ctypes as C
    import agentfield_b200 as afb
    from agentfield_b200 import _abi
    lib = _abi.load()
    master = bytes(range(0xA0, 0xC0))
    reqs = DC.random_requests(random.Random(29), 500, max_ids=6)
    for i, r in enumerate(reqs):
        r["agent_node_id"] = b"staged-node-%06d" % i
    R = packed_call(afb.ExpandedKeys(ctx), reqs, 0, master=master)
    want = DC.oracle(reqs, 0, master=master)

    def hits(pattern):
        h = C.c_uint64()
        _abi.check(lib.afc_staging_find(ctx.handle, pattern, len(pattern), C.byref(h)), ctx.handle)
        return h.value
    assert hits(b"staged-node-000123") > 0
    assert hits(master) == 0
    comps = [c for w in want for c in w["components"]]
    for c in comps[::97]:
        assert hits(c["seed"]) == 0
        assert hits(base64.urlsafe_b64encode(c["seed"]).rstrip(b"=")) == 0         # the private JWK's "d"
    for k in range(0, int(R["comp_off"][-1]), 97):
        assert hits(R["expanded"][k, :32].tobytes()) == 0 and hits(R["expanded"][k, 32:64].tobytes()) == 0
