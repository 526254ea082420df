"""The re-registration routines (agentfield_b200/csrc/afc_didrereg.cuh), compiled for the CPU (tests/hostsim/hostsim_didrereg.cpp), against
the oracle (tests/didrr_oracle.py) and the fixture: states, counts, flags, key slots and whole bodies on the golden requests and on
20 000 seeded random ones; the sizes pass against the fill pass; and afc_did_reregister_bound (libafcrypto.so, host arithmetic only)
against the real sizes, additive over requests."""
import ctypes as C
import hashlib
import json
import os
import random
import subprocess

import numpy as np
import pytest

import didrr_cases as RC
import didrr_oracle as RR
from oracle import ref_did as RD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xFE                 # never in a body: json.Marshal writes a 0xFE byte as �
P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("didrrsim") / "libafc_didrrsim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_didrereg.cpp")])
    return C.CDLL(out)


def run(sim, requests, master=RC.MASTER, server=RC.SERVER):
    """Everything the kernels write for a batch, the bodies checked against SENTINEL-filled buffers.  The key slots' pks come from the
    oracle's seeds (OpenSSL), as the expansion kernel would write them."""
    n = len(requests)
    A = RC.pack(requests)
    m, G = int(A[3][-1] - A[3][0]), int(A[6][-1] - A[6][0])
    ms = np.frombuffer(master, dtype=np.uint8).copy()
    state, counts, body_off = np.zeros(n + 1, dtype=np.uint8), np.zeros(4 * n + 1, dtype=np.uint32), np.zeros(n + 1, dtype=np.uint64)
    seeds, paths, dids = np.zeros((2 * n + 1, 32), dtype=np.uint8), np.zeros((2 * n + 1, 48), dtype=np.uint8), np.zeros((2 * n + 1, 55), dtype=np.uint8)
    rfl, ifl = np.zeros(G + 1, dtype=np.uint8), np.zeros(m + 1, dtype=np.uint8)
    args = lambda pks, body: (P(ms), server, len(server), *[P(a) for a in A], n, pks, P(state), P(counts), P(seeds), P(paths), P(dids),  # noqa: E731
                              P(rfl), P(ifl), body, P(body_off))
    assert sim.hs_didrr_run(*args(None, None)) == 0
    total = int(body_off[n])
    pks = np.zeros((2 * n + 1, 32), dtype=np.uint8)
    for t in range(2 * n):
        if seeds[t].any():
            pks[t] = np.frombuffer(RD.public_key(seeds[t].tobytes()), dtype=np.uint8)
    body = np.full(total + 64, SENTINEL, dtype=np.uint8)
    off2 = body_off.copy()
    assert sim.hs_didrr_run(*args(P(pks), P(body))) == 0
    assert (body_off == off2).all()
    assert not (body[:total] == SENTINEL).any(), "a byte the sizes pass counted was not written"
    assert (body[total:] == SENTINEL).all(), "a byte past the counted length was written"
    bodies = [body[int(body_off[i]):int(body_off[i + 1])].tobytes() for i in range(n)]
    return {"state": state[:n], "counts": counts[:4 * n].reshape(n, 4), "seeds": seeds[:2 * n], "paths": paths[:2 * n], "dids": dids[:2 * n],
            "pks": pks[:2 * n], "reg_flags": rfl[:G], "id_flags": ifl[:m], "bodies": bodies}


def check(sim, requests):
    R = run(sim, requests)
    want = RC.oracle(requests)
    g = k = 0
    for i, (r, w) in enumerate(zip(requests, want)):
        assert R["bodies"][i] == w["body"], (i, R["bodies"][i][:400], w["body"][:400])
        assert R["state"][i] == w["state"] and list(R["counts"][i]) == w["counts"], i
        for kind, name in ((0, "reasoners"), (1, "skills")):
            for x in w["gone"][kind]:
                assert bool(R["reg_flags"][g]) == x, (i, kind)
                g += 1
            for x in w["id_flags"][kind]:
                assert R["id_flags"][k] == x, (i, kind)
                k += 1
            s, t = w["slots"][kind], 2 * i + kind
            if s is None:
                assert not R["seeds"][t].any() and not R["paths"][t].any() and not R["dids"][t].any()
            else:
                assert R["paths"][t].tobytes().rstrip(b"\0") == s["path"] and R["seeds"][t].tobytes() == s["seed"] and R["dids"][t].tobytes() == s["did"]
    return R


def test_golden_requests(sim):
    reqs = RC.golden_requests()
    want = RC.oracle(reqs)
    assert {w["state"] for w in want} == {RR.UNCHANGED, RR.REMOVED, RR.PARTIAL, RR.INVALID}
    check(sim, reqs)


def test_shared_index_takes_a_survivors_did(sim):
    reqs = [r for r in RC.golden_requests() if r["agent_node_id"] == b"collide"]
    R = check(sim, reqs)
    r2 = dict(reqs[0]["agent"]["reasoners"])[b"r2"]
    assert R["dids"][0].tobytes() == r2["did"] and R["paths"][0].tobytes().rstrip(b"\0") == r2["derivation_path"]


@pytest.mark.parametrize("seed", range(4))
def test_random_5000(sim, seed):
    check(sim, RC.random_requests(random.Random(100 + seed), 5000))


def test_long_lists(sim):
    rng = random.Random(7)
    reqs = RC.random_requests(rng, 30, max_reg=300, max_new=40)
    check(sim, reqs)


def test_fixture(sim):
    g = json.load(open(os.path.join(ROOT, "tests", "golden", "did_reregister_cases.json")))
    assert bytes.fromhex(g["master_seed"]) == RC.MASTER and bytes.fromhex(g["server_id"]) == RC.SERVER
    reqs = [RC.from_json(c["request"]) for c in g["cases"]]
    R = run(sim, reqs)
    for i, c in enumerate(g["cases"]):
        assert R["bodies"][i] == bytes.fromhex(c["body"]), c["request"]["agent_node_id"]
        assert R["state"][i] == c["state"] and list(R["counts"][i]) == c["counts"]
        for kind in range(2):
            s = c["slots"][kind]
            if s is None:
                assert not R["seeds"][2 * i + kind].any()
            else:
                assert R["dids"][2 * i + kind].tobytes().decode() == s["did"]
                assert R["paths"][2 * i + kind].tobytes().rstrip(b"\0").decode() == s["path"]
                assert hashlib.sha256(R["seeds"][2 * i + kind].tobytes()).hexdigest() == s["seed_sha256"]


def test_bound_holds_and_is_additive(sim):
    from agentfield_b200 import _abi
    lib = _abi.load()
    server = b"<\xff>" * 20

    def bound(reqs):
        A = RC.pack(reqs)
        return lib.afc_did_reregister_bound(P(A[1]), P(A[3]), P(A[5]), P(A[6]), P(A[8]), len(reqs), len(server))
    rng = random.Random(3)
    for reqs in (RC.random_requests(rng, 200, esc=0.9), RC.golden_requests()):
        bodies = run(sim, reqs, server=server)["bodies"]
        assert bound(reqs) >= sum(len(b) for b in bodies)
        assert bound(reqs) == sum(bound([r]) for r in reqs)
        for r, b in zip(reqs, bodies):
            assert bound([r]) >= len(b)
    # the bound reads only the ends of the offset arrays
    A = RC.pack(RC.golden_requests())
    n = len(RC.golden_requests())
    mid = [a.copy() for a in A]
    for k in (1, 5, 8):
        mid[k][1:-1] = 0
    assert lib.afc_did_reregister_bound(P(mid[1]), P(A[3]), P(mid[5]), P(A[6]), P(mid[8]), n, 3) == \
        lib.afc_did_reregister_bound(P(A[1]), P(A[3]), P(A[5]), P(A[6]), P(A[8]), n, 3)
    assert lib.afc_did_reregister_bound(P(A[1]), P(A[3]), P(A[5]), P(A[6]), P(A[8]), 0, 3) == 0
