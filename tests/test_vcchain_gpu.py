"""afc_vc_workflow_chain_batch[_dev] on the GPU against the oracle (tests/chain_oracle.py): the golden fixture's workflows (their issuers
mapped onto real keys) and seeded random ones through the _dev call and the host-buffer call with pageable and pinned buffers; every
body parses, and its workflow_vc.vc_document is afc_vc_issue_workflow_batch's on the same inputs and verifies through
afc_vc_verify_stored_batch; the host-buffer call in a fresh process with chunks small enough to wrap the staging ring, after which no
expanded-key half is left in staging memory; one workflow of 16 384 records whose distinct DIDs take the global-memory sort; and the
service path (VCService.get_workflow_vc_chain_batch over DIDService.did_directory, device and host mirror) body for body."""
import ctypes as C
import datetime as dt
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import chain_cases as CC
import chain_oracle as CO
import workflow_cases as WC

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASTER = bytes(range(32))


def _keys(ctx, k, base=7300):
    import agentfield_b200 as afb
    from oracle import go_hash as H
    cache = afb.ExpandedKeys(ctx)
    paths = ["m/44'/%d'/0'" % (base + a) for a in range(k)]
    dids = cache.derive(MASTER, paths)
    seeds = {d: H.derive_seed(MASTER, p) for d, p in zip(dids, paths)}
    return cache, dids, seeds


def _setup(ctx, n_random=600, seed=61):
    """(cache, dids, seeds, cases, directory dict, DIDDirectory): every workflow's issuer is one of the cache's DIDs."""
    from agentfield_b200.identity import DIDDirectory
    cache, dids, seeds = _keys(ctx, 4)
    real = [d.encode() for d in dids]
    cases = CC.fixture_cases()
    for k, c in enumerate(cases):
        if c["cols"][2]:
            c["cols"][2] = real[k % len(real)]
    pool = CC.random_dids() + real
    rng = np.random.default_rng(seed)
    for i in range(n_random):
        c = CC.random_case(rng, 100 + i, pool)
        c["cols"][2] = real[int(rng.integers(len(real)))]
        cases.append(c)
    d = CC.directory([x for x in pool if x.startswith(b"did:key:zR")])
    d.update({x: cache.public_key(x.decode()) for x in real})
    pks, buf, off = CC.pack_directory(d)
    directory = DIDDirectory(list(d), list(d.values()), ctx=ctx)
    return cache, dids, seeds, cases, d, directory


def _ki(cache, dids, cases):
    return cache.key_index([c["cols"][2].decode() if c["cols"][2] else dids[0] for c in cases])


def _issued(cache, dids, cases):
    docs, off, pv, state, _ = cache.issue_workflow_packed(_ki(cache, dids, cases), *WC.pack([CO.issue_case(c) for c in cases]))
    b = docs.tobytes()
    return [(b[int(off[i]):int(off[i + 1])], pv[i].tobytes().decode(), int(state[i])) for i in range(len(cases))]


def _split(bodies, off, state):
    b = bodies.tobytes() if hasattr(bodies, "tobytes") else bytes(bodies)
    return [(int(state[i]), b[int(off[i]):int(off[i + 1])]) for i in range(len(state))]


def _host(cache, dids, directory, cases, pinned=False):
    from agentfield_b200 import _abi
    arrays = CC.pack(cases)
    ki = _ki(cache, dids, cases)
    keep = []
    if pinned:
        lib = _abi.load()

        def pin(a):
            p = lib.afc_alloc_pinned(max(a.nbytes, 1))
            h = np.frombuffer((C.c_uint8 * max(a.nbytes, 1)).from_address(p), dtype=np.uint8)[:a.nbytes].view(a.dtype).reshape(a.shape)
            h[...] = a
            keep.append(p)
            return h
        arrays = tuple(pin(a) for a in arrays)
        ki = pin(ki)
    try:
        return _split(*cache.workflow_chain_packed(directory, ki, *arrays))
    finally:
        for p in keep:
            _abi.load().afc_free_pinned(p)


def _dev(ctx, cache, dids, directory, cases):
    import torch
    dev = torch.device("cuda", ctx.device)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a.view(np.int64) if a.dtype == np.uint64 else a)).to(dev)
    d_arrays = [t(a) for a in CC.pack(cases)]
    d_ki = t(_ki(cache, dids, cases).view(np.int32))
    bodies, off, state = cache.workflow_chain_dev(directory, d_ki, d_arrays, len(cases))
    torch.cuda.synchronize(dev)
    return _split(bodies.cpu().numpy(), off.cpu().numpy(), state.cpu().numpy())


def _expected(cache, dids, cases, d):
    out = []
    for c, (doc, pv, st) in zip(cases, _issued(cache, dids, cases)):
        if CO.is_host(c, d):
            out.append((1, b""))
        else:
            assert st == 0
            out.append((0, CO.chain_body(c, d, doc=doc, proof_value=pv)))
    return out


def test_dev_and_host_buffer_calls_equal_the_oracle(ctx):
    from agentfield_b200 import _abi
    from agentfield_b200.identity import KeySet
    cache, dids, seeds, cases, d, directory = _setup(ctx)
    want = _expected(cache, dids, cases, d)
    assert sum(st == 0 for st, _ in want) > 150 and sum(st == 1 for st, _ in want) > 50
    dev = _dev(ctx, cache, dids, directory, cases)
    assert dev == want
    assert _host(cache, dids, directory, cases) == want
    assert _host(cache, dids, directory, cases, pinned=True) == want
    issued = _issued(cache, dids, cases)
    docs = []
    for (st, body), c, (doc, pv, _) in zip(dev, cases, issued):
        if st:
            continue
        v = json.loads(body)
        assert v["workflow_vc"]["vc_document"] == json.loads(doc)
        assert body.count(b'"vc_document":' + doc + b',"signature":"' + pv.encode() + b'"') == 1
        if c["cols"][2] in [x.encode() for x in dids]:
            docs.append(doc)
        if c["cols"][2].decode() in seeds and c is not cases[0]:
            assert (doc, pv) == WC.oracle_signed(CO.issue_case(c), seeds[c["cols"][2].decode()])
    ks = KeySet([cache.public_key(x) for x in dids], ctx, dids=dids)
    st, _ = ks.verify_stored(_abi.DOC_WORKFLOW_VC, docs)
    assert len(docs) > 150 and all(s == _abi.VC_VALID for s in st)


def test_empty_batch(ctx):
    cache, dids, _, _, _, directory = _setup(ctx, n_random=0)
    assert cache.workflow_chains([], directory) == []
    assert _dev(ctx, cache, dids, directory, []) == []


def test_long_workflow_takes_the_global_sort(ctx):
    """16 384 records, each with its own caller and target: 32 769 distinct DIDs, far more than one CTA sorts in shared memory."""
    from agentfield_b200.identity import DIDDirectory
    cache, dids, seeds = _keys(ctx, 2, base=7400)
    n = 16_384
    recs = [CC.record(b"vc-%05d" % k, sec=CC.T0 + k % 50, nsec=k, caller=b"did:key:zC%05d" % (n - k), target=b"did:key:zT%05d" % k,
                      issuer=dids[0].encode()) for k in range(n)]
    case = CC.workflow(0, recs, issuer=dids[0].encode())
    others = [CC.workflow(1, [CC.record(b"vc-a", caller=b"did:key:zC00001")], issuer=dids[1].encode()), CC.workflow(2, [], issuer=dids[1].encode())]
    cases = [others[0], case, others[1]]
    d = {x: CC.pk_of(x) for r in recs for x in (r["cols"][6], r["cols"][7])}
    d.update({x.encode(): cache.public_key(x) for x in dids})
    directory = DIDDirectory(list(d), list(d.values()), ctx=ctx)
    want = _expected(cache, dids, cases, d)
    assert want[1][0] == 0 and want[1][1].count(b'"resolved_from"') == 2 * n + 1
    assert _dev(ctx, cache, dids, directory, cases) == want
    assert _host(cache, dids, directory, cases) == want


def ring_main():
    """Run in a fresh process with AFC_CHUNK_ITEMS=7: the host-buffer call wraps the staging ring; then no expanded-key half is left."""
    from agentfield_b200 import _abi
    from agentfield_b200.crypto import Context
    ctx = Context(0)
    cache, dids, seeds, cases, d, directory = _setup(ctx, n_random=120, seed=62)
    want = _expected(cache, dids, cases, d)
    assert _host(cache, dids, directory, cases) == want
    assert _host(cache, dids, directory, cases, pinned=True) == want
    lib = _abi.load()
    for x in dids:
        exp = cache._expanded[cache.key_index([x])[0]].tobytes()
        for half in (exp[:32], exp[32:64]):
            h = C.c_uint64()
            _abi.check(lib.afc_staging_find(ctx.handle, half, len(half), C.byref(h)), ctx.handle)
            assert h.value == 0
    print("ok")


def test_host_buffer_call_wraps_the_ring_and_leaves_no_key():
    script = "import sys; sys.path[:0] = [sys.argv[1], sys.argv[1] + '/tests']; import test_vcchain_gpu as T; T.ring_main()"
    env = dict(os.environ, AFC_CHUNK_ITEMS="7", AFC_MIN_CHUNK_ITEMS="7")
    r = subprocess.run([sys.executable, "-c", script, ROOT], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "ok\n" in r.stdout[-20:], r.stdout[-3000:] + r.stderr[-3000:]


def _service_case(w):
    """A workflow dict of VCService.get_workflow_vc_chain_batch as a chain_oracle case."""
    enc = lambda v: v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)
    zone = lambda t: int(t.utcoffset().total_seconds())
    unix = lambda t: (t - dt.datetime(1970, 1, 1, tzinfo=dt.timezone.utc)) // dt.timedelta(seconds=1)
    evs = w["execution_vcs"]
    recs = []
    for v in evs:
        flags = (CO.AGENT_NIL if v["agent_node_id"] is None else 0) | (CO.NAME_NIL if v["workflow_name"] is None else 0) | \
            (CO.DOC_NIL if v["vc_document"] is None else 0)
        recs.append({"vc_id": enc(v["vc_id"]), "status": enc(v["status"]), "sec": unix(v["created_at"]), "nsec": v["created_at"].microsecond * 1000,
                     "zone": zone(v["created_at"]), "cols": [enc(v.get(k) or b"") for k in CO.REC_COLUMNS], "flags": flags,
                     "doc_size": v["document_size_bytes"]})
    issuer = evs[0]["issuer_did"] if evs else w["root_did"]
    cols = [enc(x) for x in (w["workflow_id"], evs[0]["session_id"] if evs else "", issuer, w["vc_id"], w["issuance_date"], w["snapshot_time"],
                             w["proof_created"])]
    s = w["snapshot"]
    return {"cols": cols, "records": recs, "wf_vc_id": enc(w["workflow_vc_id"]), "resolved_at": enc(w["resolved_at"]),
            "clock": (unix(s), s.microsecond * 1000, zone(s))}


def test_service_path_equals_the_oracle(ctx):
    """VCService.get_workflow_vc_chain_batch over a DIDService registry (DIDService.did_directory): workflows as dicts with aware datetimes in
    several zones and None fields, built by the device or, where it declines (a document nested 40 deep, a long resolved_at), by the host
    mirror, in request order; a workflow without records is issued under the root DID, whose member the bundle holds.  A document Go cannot
    marshal raises ValueError."""
    import agentfield_b200 as afb
    from agentfield_b200 import _abi, services
    from oracle import go_hash as H
    cache = afb.ExpandedKeys(ctx)
    didsvc = services.DIDService(cache, MASTER, b"chain-server")
    didsvc.register_agents_batch([{"agent_node_id": "agent-%d" % a, "reasoners": ["r%d" % k for k in range(3)], "skills": ["s0"]} for a in range(4)])
    directory = didsvc.did_directory()
    root = didsvc.root_did
    paths = {root: services.DIDService.ROOT_PATH}
    comps = []
    for a in didsvc.agent_nodes.values():
        for e in [a] + list(a["reasoners"].values()) + list(a["skills"].values()):
            paths[e["did"]] = e["derivation_path"]
            comps.append(e["did"])
    keys = dict(zip(directory.dids, directory.pks))
    assert root.encode() in keys and len(keys) == len(paths)
    svc = services.VCService(cache)
    rng = np.random.default_rng(63)
    zones = [dt.timezone.utc, dt.timezone(dt.timedelta(hours=5, minutes=30)), dt.timezone(dt.timedelta(hours=-8))]
    deep = b"[" * 40 + b"]" * 40
    docs = [b'{"a": 1, "h": "<b>&"}', None, b'"x"', b" [ 1 , 2 ] "]
    wfs = []
    for i in range(60):
        evs = []
        for k in range(int(rng.integers(0, 7))) if i else []:
            t = dt.datetime(2026, 9, 21, 6, 0, int(rng.integers(60)), int(rng.choice([0, 500000, int(rng.integers(10 ** 6))])),
                            tzinfo=dt.timezone.utc).astimezone(zones[int(rng.integers(3))])
            doc = deep if (i % 17 == 5 and k == 0) else docs[int(rng.integers(len(docs)))]
            evs.append({"vc_id": "vc-%d-%d" % (i, k), "execution_id": "exec-%d-%d" % (i, k), "workflow_id": "wf-%d" % i, "session_id": "sess-%d" % i,
                        "agent_node_id": None if k % 3 == 1 else "agent-%d" % (k % 4), "workflow_name": None if k % 2 else "",
                        "issuer_did": comps[int(rng.integers(len(comps)))], "target_did": comps[int(rng.integers(len(comps)))],
                        "caller_did": "" if k % 4 == 3 else comps[int(rng.integers(len(comps)))], "vc_document": doc, "signature": "sig",
                        "storage_uri": "", "document_size_bytes": 0 if doc is None else len(doc), "input_hash": "ih", "output_hash": "oh",
                        "status": ["succeeded", "failed", "running", " Done "][int(rng.integers(4))], "created_at": t})
        wfs.append({"workflow_id": "wf-%d" % i, "execution_vcs": evs, "root_did": root, "vc_id": "wvc-doc-%d" % i, "workflow_vc_id": "wvc-%d" % i,
                    "issuance_date": "2026-09-21T06:01:00Z", "snapshot_time": "2026-09-21T06:01:00Z", "proof_created": "2026-09-21T06:01:00Z",
                    "resolved_at": "2026-09-21T06:01:00Z" + ("x" * 60 if i % 13 == 7 else ""),
                    "snapshot": dt.datetime(2026, 9, 21, 6, 1, 0, 250000, tzinfo=zones[i % 3])})
    states = [st for st, _ in cache.workflow_chains(wfs, directory)]
    assert states.count(_abi.CHAIN_HOST) >= 6 and states.count(_abi.CHAIN_BUILT) >= 40
    got = svc.get_workflow_vc_chain_batch(wfs, directory)
    assert len(got) == len(wfs)
    for w, body in zip(wfs, got):
        case = _service_case(w)
        issuer = case["cols"][2].decode()
        _, pv = WC.oracle_signed(CO.issue_case(case), H.derive_seed(MASTER, paths[issuer]))
        assert body == CO.chain_body(case, keys, proof_value=pv), w["workflow_id"]
        json.loads(body)
    assert b'"did_resolution_bundle":{"' + root.encode() + b'":{"method":"key"' in got[0]       # no records: the root DID issues
    w = next(w for w in wfs if w["execution_vcs"])
    with pytest.raises(ValueError):
        svc.get_workflow_vc_chain_batch([dict(w, execution_vcs=[dict(w["execution_vcs"][0], vc_document=b"{")])], directory)
