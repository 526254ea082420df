"""The DID resolution routines (agentfield_b200/csrc/afc_didresolve.cuh), compiled for the CPU (tests/hostsim/hostsim_didresolve.cpp),
against the oracle (tests/resolve_oracle.py): the golden fixture and 20 000 seeded random requests.  Also checks that the sizes pass and
the emit pass agree, that the canonical JWK texts written at attach are the oracle's, and that the bound's per-request terms cover every
body (afc_did_resolve_bound adds them up over requests; tests/c_abi/did_resolve.c checks the library's sum)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import resolve_cases as RC
import resolve_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xFE


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("dressim") / "libafc_dressim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_didresolve.cpp")])
    lib = C.CDLL(out)
    lib.hs_dres_request_fixed.restype = C.c_uint64
    return lib


class Buf:
    """bytes in a buffer padded past their end (the word reads of ByteWindow may touch up to 3 bytes beyond)."""

    def __init__(self, b):
        self.n = len(b)
        self.a = np.frombuffer(bytes(b) + bytes(8), dtype=np.uint8).copy()

    @property
    def p(self):
        return self.a.ctypes.data_as(C.c_void_p)


class Directory:
    """A registry's directory through the attach routine: each entry's lengths and side text, and the largest body."""

    def __init__(self, hs, reg):
        self.entries = RC.directory_entries(reg)
        self.index = {e["did"]: k for k, e in enumerate(self.entries)}
        self.info = []
        for e in self.entries:
            cols = [Buf(e[k]) for k in ("did", "derivation_path", "function_name", "public_key_jwk")]
            out = (C.c_uint32 * 3)()
            hs.hs_dres_entry(e["kind"], *[x for c in cols for x in (c.p, C.c_uint64(c.n))], out, None)
            side = b""
            if out[2]:
                sb = np.full(out[2] + 32, SENTINEL, dtype=np.uint8)
                hs.hs_dres_entry(e["kind"], *[x for c in cols for x in (c.p, C.c_uint64(c.n))], out, sb.ctypes.data_as(C.c_void_p))
                assert (sb[out[2]:] == SENTINEL).all()
                side = sb[:out[2]].tobytes()
            self.info.append((cols, out[0], out[1], Buf(side)))
        self.largest = max([max(i[1], i[2]) for i in self.info] + [0])

    def run(self, hs, kind, req):
        """(state, body): the buffer starts as SENTINEL bytes, and the emit pass must write exactly the length the sizes pass reported."""
        k = self.index.get(req) if req else None
        cols, rlen, dlen, side = self.info[k] if k is not None else ([Buf(b"")] * 4, 0, 0, Buf(b""))
        r = Buf(req)
        args = [kind, r.p, C.c_uint64(r.n), int(k is not None), self.entries[k]["kind"] if k is not None else 0]
        args += [x for c in cols for x in (c.p, C.c_uint64(c.n))] + [side.p, C.c_uint64(side.n), rlen, dlen]
        state, n = C.c_uint32(), C.c_uint64()
        hs.hs_dres_request(*args, C.byref(state), None, C.byref(n))
        body = np.full(n.value + 32, SENTINEL, dtype=np.uint8)
        state2, n2 = C.c_uint32(), C.c_uint64()
        hs.hs_dres_request(*args, C.byref(state2), body.ctypes.data_as(C.c_void_p), C.byref(n2))
        assert (state2.value, n2.value) == (state.value, n.value)
        assert (body[n.value:] == SENTINEL).all(), "the emit pass wrote past the length the sizes pass reported"
        return state.value, body[:n.value].tobytes()


@pytest.fixture(scope="module")
def fixture(hs):
    reg, reqs, expected = RC.load_fixture()
    return reg, reqs, expected, Directory(hs, reg)


def test_fixture_is_the_oracles(fixture):
    reg, reqs, expected, _ = fixture
    fresh = RC.fixture_registry()
    assert RC.registry_to_json(fresh) == RC.registry_to_json(reg)
    for (k, d), outs in zip(reqs, expected):
        assert [tuple(o) for o in RC.outcomes_json(RO.outcomes(reg, k, d))] == outs


def test_fixture_requests(hs, fixture):
    reg, reqs, expected, D = fixture
    states = []
    for (k, d), outs in zip(reqs, expected):
        st, body = D.run(hs, k, d)
        assert RC.accepts_stored(outs, st, body), (k, d[:60], st, body[:200])
        states.append(st)
    assert {0, 1, 2, 3} <= set(states)


def test_named_cases(hs, fixture):
    reg, _, _, D = fixture
    root = reg["root_did"]
    st, body = D.run(hs, RO.RESOLVE, root)
    assert st == 0 and b'"component_type":"agentfield_server","derivation_path":"m/44\'/0\'"' in body and b'"function_name":""' in body
    assert D.run(hs, RO.RESOLVE, b"") == (2, b'{"error":"DID parameter is required"}')
    assert D.run(hs, RO.RESOLVE, b"did:key:zNone") == (1, b'{"error":"DID not found"}')
    assert D.run(hs, RO.DOCUMENT, b"did:\xff<") == (1, b'{"details":"DID not found: did:\\ufffd\\u003c","error":"DID not found"}')
    assert D.run(hs, 7, root)[0] == 3                             # an unknown kind goes to the host
    by_jwk = {e["public_key_jwk"]: e["did"] for e in D.entries if e["kind"] == RO.AGENT}
    assert D.run(hs, RO.DOCUMENT, by_jwk[b"null"])[1].count(b'"publicKeyJwk":null,') == 1
    for jwk in (b"[1,2]", b"", b'{"a":1,"a":2}', b'{"huge":1e400}'):
        assert D.run(hs, RO.DOCUMENT, by_jwk[jwk])[0] == 3, jwk[:20]
        assert D.run(hs, RO.RESOLVE, by_jwk[jwk])[0] == 0
    padded = by_jwk[b'{"pad":"' + b"x" * 4000 + b'"}']             # both bodies over the cap
    assert D.run(hs, RO.DOCUMENT, padded)[0] == 3 and D.run(hs, RO.RESOLVE, padded)[0] == 3


def test_side_texts_are_canonical(fixture):
    _, _, _, D = fixture
    sides = 0
    for e, (_, _, dlen, side) in zip(D.entries, D.info):
        if not dlen:
            continue
        ok, text, exact = RO.jwk_marshal(e["public_key_jwk"])
        assert ok and exact and text is not None
        if side.n:
            sides += 1
            assert side.a[:side.n].tobytes() == text != e["public_key_jwk"]
        else:
            assert e["public_key_jwk"] == text
    assert sides >= 3


def test_random_requests_match_the_oracle(hs, fixture):
    reg, _, _, D = fixture
    rng = np.random.default_rng(0xD1D)
    for k, d in RC.random_requests(reg, rng, 20000):
        st, body = D.run(hs, k, d)
        assert RO.accepts(RO.outcomes(reg, k, d), st, body), (k, d, st, body[:200])


def test_bound_terms_cover_every_body(hs, fixture):
    reg, reqs, _, D = fixture
    per = max(D.largest, hs.hs_dres_request_fixed())
    assert D.largest <= RO.CAP
    rng = np.random.default_rng(7)
    for k, d in reqs + RC.random_requests(reg, rng, 2000):
        _, body = D.run(hs, k, d)
        assert len(body) <= per + 6 * len(d)
