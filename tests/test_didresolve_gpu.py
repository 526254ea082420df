"""afc_did_resolve_batch[_dev] on the GPU against the oracle (tests/resolve_oracle.py): the golden fixture and seeded random batches
through the _dev call and the host-buffer call (pageable and pinned buffers); the host-buffer call in a fresh process with chunks small
enough to wrap the staging ring; a directory of 2^20 DIDs checked on a sample; DIDService.serve_did_requests after registrations and a
re-registration that gives two components one DID; and afc_vc_workflow_chain_batch giving the same bytes on a directory with identities
as on one without."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import resolve_cases as RC
import resolve_oracle as RO

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASTER = bytes(range(32))


def directory_of(ctx, reg):
    """The registry's directory with identities (each DID's first holder in registration order; keys are not read by these calls)."""
    from agentfield_b200.identity import DIDDirectory
    ents = RC.directory_entries(reg)
    d = DIDDirectory([e["did"] for e in ents], [bytes(32)] * len(ents), ctx=ctx)
    d.set_identities(*[[e[k] for e in ents] for k in ("kind", "derivation_path", "function_name", "public_key_jwk")])
    return d


def host_call(directory, requests, pinned=False):
    from agentfield_b200 import _abi
    kinds, reqs, off = directory.pack_requests(requests)
    keep = []
    if pinned:
        lib = _abi.load()

        def pin(a):
            p = lib.afc_alloc_pinned(max(a.nbytes, 1))
            h = np.frombuffer((C.c_uint8 * max(a.nbytes, 1)).from_address(p), dtype=np.uint8)[:a.nbytes].view(a.dtype)
            h[...] = a
            keep.append(p)
            return h
        kinds, reqs, off = pin(kinds), pin(reqs), pin(off)
    try:
        bodies, body_off, state = directory.resolve_packed(kinds, reqs, off)
        b = bodies.tobytes()
        return [(int(state[i]), b[int(body_off[i]):int(body_off[i + 1])]) for i in range(len(requests))]
    finally:
        for p in keep:
            _abi.load().afc_free_pinned(p)


def dev_call(ctx, directory, requests):
    import torch
    dev = torch.device("cuda", ctx.device)
    kinds, reqs, off = directory.pack_requests(requests)
    bodies, body_off, state = directory.resolve_dev(torch.from_numpy(kinds).to(dev), torch.from_numpy(reqs).to(dev),
                                                    torch.from_numpy(off.view(np.int64)).to(dev), len(requests))
    torch.cuda.synchronize(dev)
    b, o, s = bodies.cpu().numpy().tobytes(), body_off.cpu().numpy(), state.cpu().numpy()
    return [(int(s[i]), b[int(o[i]):int(o[i + 1])]) for i in range(len(requests))]


def test_fixture_through_both_calls(ctx):
    reg, reqs, expected = RC.load_fixture()
    directory = directory_of(ctx, reg)
    for got in (dev_call(ctx, directory, reqs), host_call(directory, reqs), host_call(directory, reqs, pinned=True)):
        for (k, d), outs, (st, body) in zip(reqs, expected, got):
            assert RC.accepts_stored(outs, st, body), (k, d[:60], st, body[:200])
        assert {0, 1, 2, 3} <= {st for st, _ in got}


def test_random_batches(ctx):
    reg = RC.fixture_registry()
    directory = directory_of(ctx, reg)
    rng = np.random.default_rng(0x5E5)
    for n in (1, 129, 5000):
        reqs = RC.random_requests(reg, rng, n)
        dev = dev_call(ctx, directory, reqs)
        assert dev == host_call(directory, reqs)
        for (k, d), (st, body) in zip(reqs, dev):
            assert RO.accepts(RO.outcomes(reg, k, d), st, body), (k, d, st, body[:200])
    assert directory.resolve([]) == [] and dev_call(ctx, directory, []) == []


def ring_main():
    """Run in a fresh process with AFC_CHUNK_ITEMS=7: the host-buffer call runs many chunks around the staging ring."""
    from agentfield_b200.crypto import Context
    ctx = Context(0)
    reg = RC.fixture_registry()
    directory = directory_of(ctx, reg)
    reqs = RC.random_requests(reg, np.random.default_rng(11), 300)
    got = host_call(directory, reqs)
    assert got == host_call(directory, reqs, pinned=True)
    for (k, d), (st, body) in zip(reqs, got):
        assert RO.accepts(RO.outcomes(reg, k, d), st, body), (k, d, st, body[:200])
    print("ok")


def test_host_buffer_call_wraps_the_ring():
    script = "import sys; sys.path[:0] = [sys.argv[1], sys.argv[1] + '/tests']; import test_didresolve_gpu as T; T.ring_main()"
    env = dict(os.environ, AFC_CHUNK_ITEMS="7", AFC_MIN_CHUNK_ITEMS="7")
    r = subprocess.run([sys.executable, "-c", script, ROOT], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "ok\n" in r.stdout[-20:], r.stdout[-3000:] + r.stderr[-3000:]


def big_registry(agents=1 << 14, per_agent=63, seed=5):
    """About 2^20 DIDs: 2^14 agents with up to 63 components each, every 100th stored JWK in a non-canonical spelling."""
    rng = np.random.default_rng(seed)
    root_pk = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    out, k = [], 0
    for a in range(agents):
        def comp(tag):
            nonlocal k
            k += 1
            pk = bytes(rng.integers(0, 256, 32, dtype=np.uint8)) if k % 4096 == 0 else k.to_bytes(32, "little")
            jwk = RO.RD.public_jwk(pk)
            if k % 100 == 0:
                jwk = b" " + jwk.replace(b",", b", ")
            return {"did": RO.RD.did_key(pk), "derivation_path": b"m/44'/7'/%d'/%s" % (a, tag), "public_key_jwk": jwk}
        ag = comp(b"a")
        m = int(rng.integers(per_agent // 2, per_agent + 1))
        ag["reasoners"] = [(b"r%d" % j, dict(comp(b"0'/%d'" % j), function_name=b"r%d" % j)) for j in range(m // 2)]
        ag["skills"] = [(b"s%d" % j, dict(comp(b"1'/%d'" % j), function_name=b"s%d" % j)) for j in range(m - m // 2)]
        out.append(ag)
    return {"root_did": RO.RD.did_key(root_pk), "root_pk": root_pk, "agents": out}


def test_directory_of_a_million_dids(ctx):
    reg = big_registry()
    directory = directory_of(ctx, reg)
    n_dids = len(directory.dids)
    assert n_dids > 500_000
    rng = np.random.default_rng(3)
    pick = rng.integers(0, n_dids, 1 << 16)
    reqs = [(int(k & 1), directory.dids[int(p)] if k % 20 else b"did:key:zUnknown%d" % k) for k, p in enumerate(pick)]
    got = dev_call(ctx, directory, reqs)
    sample = rng.choice(len(reqs), 3000, replace=False)
    index = {}
    for e in RC.directory_entries(reg):
        index.setdefault(e["did"], e)
    for i in sample:
        k, d = reqs[i]
        e = index.get(d)
        assert RO.accepts([RO.outcome(k, d, e)], *got[i]), (k, d, got[i][:200])
    assert sum(st == 0 for st, _ in got) > 0.9 * len(got)


def test_service_after_registration_and_reregistration(ctx):
    import agentfield_b200 as afb
    from agentfield_b200 import _abi, services
    cache = afb.ExpandedKeys(ctx)
    svc = services.DIDService(cache, MASTER, b"resolve-server")
    svc.register_agents_batch([{"agent_node_id": "agent-%d" % a, "reasoners": ["plan", "q\"<&>"], "skills": ["s "]} for a in range(3)])
    first = svc.serve_did_requests([(_abi.DIDRES_RESOLVE, svc.root_did)])
    assert first[0][0] == 200
    # agent-1 drops "plan" and adds two reasoners: both new ones take the slot's DID
    svc.reregister_agents_batch([{"agent_node_id": "agent-1", "reasoners": ["q\"<&>", "n1", "n2"], "skills": ["s "]}])

    def reg_of(s):
        enc = lambda v: v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)
        comp = lambda c: {"did": enc(c["did"]), "derivation_path": enc(c["derivation_path"]), "public_key_jwk": enc(c["public_key_jwk"]),
                          "function_name": enc(c["function_name"])}
        agents = [{"did": enc(a["did"]), "derivation_path": enc(a["derivation_path"]), "public_key_jwk": enc(a["public_key_jwk"]),
                   "reasoners": [(enc(k), comp(c)) for k, c in a["reasoners"].items()], "skills": [(enc(k), comp(c)) for k, c in a["skills"].items()]}
                  for a in s.agent_nodes.values()]
        return {"root_did": enc(s.root_did), "root_pk": cache.public_key(s.root_did), "agents": agents}
    reg = reg_of(svc)
    dids = [e["did"] for e in RO.identities(reg)]
    dup = [d for d in set(dids) if dids.count(d) > 1]
    assert len(dup) == 1
    reqs = [(k, d) for d in list(dict.fromkeys(dids)) + [b"", b"did:key:zNope"] for k in (_abi.DIDRES_RESOLVE, _abi.DIDRES_DOCUMENT)]
    got = svc.serve_did_requests(reqs)
    for (k, d), (status, body) in zip(reqs, got):
        outs = RO.outcomes(reg, k, d)
        assert any(o[0] == status and o[1] == body for o in outs), (k, d, status, body[:200])
        cs = RO.candidates(reg, d)
        if len(cs) > 1:
            assert (status, body) == RO.outcome(k, d, cs[0])[:2]       # the first-registered holder
    assert svc.serve_did_requests([]) == []


def test_chain_bytes_do_not_depend_on_identities(ctx):
    import chain_cases as CC
    import agentfield_b200 as afb
    from agentfield_b200.identity import DIDDirectory
    cache = afb.ExpandedKeys(ctx)
    dids = cache.derive(MASTER, ["m/44'/%d'/0'" % (7500 + a) for a in range(3)])
    real = [d.encode() for d in dids]
    cases = CC.fixture_cases()
    for k, c in enumerate(cases):
        if c["cols"][2]:
            c["cols"][2] = real[k % len(real)]
    d = CC.directory()
    d.update({x: cache.public_key(x.decode()) for x in real})
    plain = DIDDirectory(list(d), list(d.values()), ctx=ctx)
    rich = DIDDirectory(list(d), list(d.values()), ctx=ctx)
    n = len(d)
    rich.set_identities([1] * n, [b"m/44'/1'"] * n, [b""] * n, [b'{"a":[1, 2]}'] * n)
    ki = cache.key_index([c["cols"][2].decode() if c["cols"][2] else dids[0] for c in cases])
    a = cache.workflow_chain_packed(plain, ki, *CC.pack(cases))
    b = cache.workflow_chain_packed(rich, ki, *CC.pack(cases))
    assert all((x == y).all() for x, y in zip(a, b)) and len(a[0]) > 1000
