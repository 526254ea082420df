"""The DID-registration routines (agentfield_b200/csrc/afc_didreg.cuh), compiled for the CPU (tests/hostsim/hostsim_didreg.cpp), against
the oracle (oracle/ref_did.py) and the fixture: FNV-1a, path text at the index extremes, the table-free base64url, shadowing and ranks on
heavily repeated lists, derived seeds, whole bodies; the sizes pass against the fill pass, and afc_did_register_bound (libafcrypto.so, host
arithmetic only) against the real sizes."""
import base64
import ctypes as C
import hashlib
import json
import os
import random
import subprocess

import numpy as np
import pytest

import did_cases as DC
from oracle import ref_did as RD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xFE                 # never in a body: json.Marshal writes a 0xFE byte as �
P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("didrsim") / "libafc_didrsim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_didreg.cpp")])
    lib = C.CDLL(out)
    lib.hs_didr_fnv1a.restype = C.c_uint32
    lib.hs_didr_server_hash.restype = C.c_uint32
    return lib


def run(sim, requests, agent_base=0, master=DC.MASTER, server=DC.SERVER):
    """Everything the kernels write for a batch, the bodies checked against SENTINEL-filled buffers: (comp_off, id_flags, id_rank, seeds,
    paths, dids, kept, bodies).  pks come from the oracle's seeds (OpenSSL), as the expansion kernel would write them."""
    n = len(requests)
    nodes, node_off, id_idx, ids, id_off = DC.pack(requests)
    m = int(id_idx[-1])
    S = n + m
    ai = np.arange(agent_base, agent_base + n, dtype=np.uint64).astype(np.uint32)
    ms = np.frombuffer(master, dtype=np.uint8).copy()
    comp_off, body_off = np.zeros(n + 1, dtype=np.uint64), np.zeros(n + 1, dtype=np.uint64)
    fl, rk = np.zeros(m + 1, dtype=np.uint8), np.zeros(m + 1, dtype=np.uint32)
    seeds, paths = np.zeros((S + 1, 32), dtype=np.uint8), np.zeros((S + 1, 48), dtype=np.uint8)
    dids, kept = np.zeros((S + 1, 55), dtype=np.uint8), np.zeros(S + 1, dtype=np.uint8)
    args = lambda pks, body: (P(ms), server, len(server), P(nodes), P(node_off), P(ai), P(id_idx), P(ids), P(id_off), n, pks,  # noqa: E731
                              P(comp_off), P(fl), P(rk), P(seeds), P(paths), P(dids), P(kept), body, P(body_off))
    assert sim.hs_didr_run(*args(None, None)) == 0
    total = int(body_off[n])
    C_ = int(comp_off[n])
    pks = np.zeros((S + 1, 32), dtype=np.uint8)
    for c in range(C_):
        pks[c] = np.frombuffer(RD.public_key(seeds[c].tobytes()), dtype=np.uint8)
    body = np.full(total + 64, SENTINEL, dtype=np.uint8)
    off2 = body_off.copy()
    assert sim.hs_didr_run(*args(P(pks), P(body))) == 0
    assert (body_off == off2).all()
    assert not (body[:total] == SENTINEL).any(), "a byte the sizes pass counted was not written"
    assert (body[total:] == SENTINEL).all(), "a byte past the counted length was written"
    bodies = [body[int(body_off[i]):int(body_off[i + 1])].tobytes() for i in range(n)]
    return comp_off, fl[:m], rk[:m], seeds[:S], paths[:S], dids[:S], kept[:S], bodies


def check(sim, requests, agent_base=0):
    comp_off, _, _, seeds, paths, dids, kept, bodies = run(sim, requests, agent_base)
    want = DC.oracle(requests, agent_base)
    for i, w in enumerate(want):
        assert bodies[i] == w["body"], (i, bodies[i][:300], w["body"][:300])
        c0, c1 = int(comp_off[i]), int(comp_off[i + 1])
        assert c1 - c0 == len(w["components"])
        for c, wc in zip(range(c0, c1), w["components"]):
            assert paths[c].tobytes().rstrip(b"\0") == wc["path"] and paths[c][len(wc["path"]):].sum() == 0
            assert seeds[c].tobytes() == wc["seed"]
            assert dids[c].tobytes() == wc["did"]
            assert bool(kept[c]) == wc["kept"]
    C_ = int(comp_off[-1])
    assert not seeds[C_:].any() and not paths[C_:].any() and not dids[C_:].any() and not kept[C_:].any()
    return bodies


def test_fnv1a_vectors(sim):
    for s, h in ((b"", 0x811C9DC5), (b"a", 0xE40C292C), (b"foobar", 0xBF9CF968)):
        assert sim.hs_didr_fnv1a(s, len(s)) == h
    rng = random.Random(1)
    for _ in range(2000):
        s = bytes(rng.randrange(256) for _ in range(rng.randrange(40)))
        assert sim.hs_didr_fnv1a(s, len(s)) == RD.fnv1a32(s)
        assert sim.hs_didr_server_hash(s, len(s)) == RD.server_hash(s)


@pytest.mark.parametrize("h", [0, 1, 9, 10, 2 ** 31 - 1])
@pytest.mark.parametrize("a", [0, 10, 99, 2 ** 31 - 1, 2 ** 32 - 1])
def test_path_text(sim, h, a):
    out = np.zeros(64, dtype=np.uint8)
    for kind in range(3):
        for j in (0, 9, 10, 1000, 2 ** 32 - 1):
            L = sim.hs_didr_path(kind, h, a, j, P(out))
            want = RD.agent_path(h, a) if kind == 0 else RD.component_path(h, a, kind - 1, j)
            assert L == len(want) and out[:L].tobytes() == want and L <= 44


def test_base64url_without_table(sim):
    rng = np.random.default_rng(7)
    edge = [bytes([v] * 32) for v in (0, 0xFF, 0xFB, 0xFC, 0xF8, 0x3E, 0x3F, 0xBE)] + [bytes(range(32)), bytes(range(224, 256))]
    data = np.concatenate([np.frombuffer(b"".join(edge), dtype=np.uint8).reshape(-1, 32), rng.integers(0, 256, (100000, 32), dtype=np.uint8)])
    out = np.zeros((len(data), 43), dtype=np.uint8)
    sim.hs_didr_b64_32(P(data), len(data), P(out))
    for k in list(range(len(edge))) + list(rng.integers(0, len(data), 5000)):
        assert out[k].tobytes() == base64.urlsafe_b64encode(data[k].tobytes()).rstrip(b"=")
    # every character of the alphabet, and the whole batch at once
    want = np.frombuffer(b"".join(base64.urlsafe_b64encode(d.tobytes())[:43] for d in data), dtype=np.uint8).reshape(-1, 43)
    assert (out == want).all()
    did = np.zeros(55, dtype=np.uint8)
    for d in data[:200]:
        sim.hs_didr_did(P(d), P(did))
        assert did.tobytes() == RD.did_key(d.tobytes())


def test_identity_sizes(sim):
    counted, arith = C.c_uint64(), C.c_uint64()
    for kind in range(3):
        for ident in [b"", b"x", b"summarize_text_17"] + DC.ESCAPES:
            for a, j in ((0, 0), (2 ** 32 - 1, 2 ** 32 - 1), (123, 45)):
                sim.hs_didr_entry_bytes(kind, 2 ** 31 - 1, a, j, ident, len(ident), C.byref(counted), C.byref(arith))
                assert counted.value == arith.value


@pytest.mark.parametrize("seed", range(6))
def test_shadowing_and_ranks_random(sim, seed):
    rng = random.Random(seed)
    reqs = DC.random_requests(rng, 40, max_ids=30, dup=0.7, alphabet=3)
    _, fl, rk, *_ = run(sim, reqs)
    _, _, id_idx, _, _ = DC.pack(reqs)
    flat = [x for r in reqs for x in list(r["reasoners"]) + list(r["skills"])]
    for L in range(2 * len(reqs)):
        lo, hi = int(id_idx[L]), int(id_idx[L + 1])
        lst = flat[lo:hi]
        kept_keys = sorted(set(x for x in lst if x))
        for k in range(lo, hi):
            x = flat[k]
            if not x:
                assert fl[k] == 0
                continue
            shadowed = x in lst[k - lo + 1:]
            assert fl[k] == (3 if shadowed else 1)
            if not shadowed:
                assert rk[k] == kept_keys.index(x)


def test_bodies_random(sim):
    rng = random.Random(11)
    check(sim, DC.random_requests(rng, 300, max_ids=10), agent_base=5)


def test_bodies_edge(sim):
    check(sim, DC.golden_requests())
    check(sim, [{"agent_node_id": b"", "reasoners": [b""] * 5, "skills": [b""] * 3}], agent_base=2 ** 32 - 1)
    check(sim, [{"agent_node_id": b"n", "reasoners": [b"r"], "skills": []}], agent_base=0)


def test_fixture(sim):
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "did_register_cases.json")))
    reqs = [{"agent_node_id": bytes.fromhex(c["agent_node_id"]), "reasoners": [bytes.fromhex(x) for x in c["reasoners"]],
             "skills": [bytes.fromhex(x) for x in c["skills"]]} for c in g["cases"]]
    assert bytes.fromhex(g["master_seed"]) == DC.MASTER and bytes.fromhex(g["server_id"]) == DC.SERVER
    comp_off, _, _, seeds, paths, dids, kept, bodies = run(sim, reqs, g["agent_base"])
    for i, c in enumerate(g["cases"]):
        assert bodies[i] == bytes.fromhex(c["body"])
        c0 = int(comp_off[i])
        for k, wc in enumerate(c["components"]):
            assert paths[c0 + k].tobytes().rstrip(b"\0").decode() == wc["path"]
            assert dids[c0 + k].tobytes().decode() == wc["did"]
            assert hashlib.sha256(seeds[c0 + k].tobytes()).hexdigest() == wc["seed_sha256"]


def test_bound_holds_on_escape_heavy_inputs(sim):
    from agentfield_b200 import _abi
    lib = _abi.load()
    rng = random.Random(3)
    worst = [b"\x01" * 40, b"<" * 33, b"\xff" * 50, b"\xe2\x80\xa8" * 10]
    for reqs in (DC.random_requests(rng, 50, esc=0.9), [{"agent_node_id": b"\x00" * 64, "reasoners": worst * 4, "skills": worst}],
                 [{"agent_node_id": b"a", "reasoners": [b"q%d" % k for k in range(300)], "skills": []}]):
        server = b"<\xff>" * 20
        *_, bodies = run(sim, reqs, 2 ** 32 - 300, server=server)
        nodes, node_off, id_idx, ids, id_off = DC.pack(reqs)
        bound = lib.afc_did_register_bound(P(node_off), P(id_idx), P(id_off), len(reqs), len(server))
        assert bound >= sum(len(b) for b in bodies)
        for i in range(len(reqs)):                                 # additive: each request within its own bound
            one = DC.pack([reqs[i]])
            *_, b1 = run(sim, [reqs[i]], 2 ** 32 - 1, server=server)
            assert lib.afc_did_register_bound(P(one[1]), P(one[2]), P(one[4]), 1, len(server)) >= len(b1[0])
