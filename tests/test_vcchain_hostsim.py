"""The workflow-chain routines (agentfield_b200/csrc/afc_vcchain.cuh), compiled for the CPU (tests/hostsim/hostsim_vcchain.cpp), against
the oracle (tests/chain_oracle.py): the golden fixture's bodies and states, 10 000 seeded random workflows, Time.MarshalJSON over zones
and nanoseconds, the bundle's DID filter.  Also checks that the sizes pass and the emit passes agree, and that
afc_vc_workflow_chain_bound (libafcrypto.so, host arithmetic only) covers every body and is additive over workflows."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import chain_cases as CC
import chain_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xFE


@pytest.fixture(scope="module")
def vcc(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("vccsim") / "libafc_vccsim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_vcchain.cpp")])
    return C.CDLL(out)


def P(a):
    return a.ctypes.data_as(C.c_void_p)


def run(vcc, case, directory):
    """(state, body) as the kernels write one workflow; the body is None for a HOST workflow.  The buffer starts as SENTINEL bytes: the
    emit passes must write exactly the length the sizes pass reported."""
    a = CC.pack([case])
    pks, dids, doff = CC.pack_directory(directory)
    args = [P(a[0]), P(a[1]), P(a[3]), P(a[4]), P(a[5]), len(case["records"]), P(a[6]), P(a[7]), P(a[8]), P(a[9]), P(a[10]), P(a[11]), P(a[12]),
            P(a[13]), P(dids), P(doff), P(pks), len(directory)]
    state, n = C.c_uint32(), C.c_uint64()
    assert vcc.hs_vcc_chain(*args, C.byref(state), None, C.byref(n)) == 0
    if state.value == 1:
        return 1, None
    body = np.full(n.value + 32, SENTINEL, dtype=np.uint8)
    n2 = C.c_uint64()
    assert vcc.hs_vcc_chain(*args, C.byref(state), P(body), C.byref(n2)) == 0
    assert n2.value == n.value
    assert not (body[:n.value] == SENTINEL).any(), "a byte the sizes pass counted was not written"
    assert (body[n.value:] == SENTINEL).all(), "a byte past the counted length was written"
    return 0, body[:n.value].tobytes()


def bound(cases):
    from agentfield_b200 import _abi
    a = CC.pack(cases)
    return _abi.load().afc_vc_workflow_chain_bound(_abi.ptr(a[1]), _abi.ptr(a[2]), _abi.ptr(a[4]), _abi.ptr(a[7]), _abi.ptr(a[10]), len(cases))


def check(vcc, case, directory):
    state, body = run(vcc, case, directory)
    if CO.is_host(case, directory):
        assert state == 1
        return None
    assert state == 0
    assert body == CO.chain_body(case, directory)
    assert bound([case]) >= len(body)
    return body


def test_fixture(vcc):
    cases, d, expected = CC.load_fixture()
    assert len(cases) >= 16
    for c, (st, body) in zip(cases, expected):
        got_state, got = run(vcc, c, d)
        assert got_state == st
        if st == 0:
            assert got == body
            import json
            json.loads(got)
    # every case the fixture promises: omitted member, HOST decisions, raw-byte vs escaped key order
    assert b"did_resolution_bundle" not in expected[9][1] and expected[3][0] == expected[4][0] == expected[6][0] == 1
    assert expected[14][0] == 1 and expected[15][0] == 0
    b8 = expected[8][1]
    assert b8.index(b'"did:key:z\\u003cesc') < b8.index(b'"did:key:zA"')


def test_fixture_matches_the_oracle():
    cases, d, expected = CC.load_fixture()
    for c, (st, body) in zip(cases, expected):
        assert st == (1 if CO.is_host(c, d) else 0)
        if st == 0:
            assert body == CO.chain_body(c, d)


def test_random_workflows(vcc):
    rng = np.random.default_rng(77)
    dids = CC.random_dids()
    d = CC.directory([x for x in dids if x.startswith(b"did:key:zR")])
    built = host = 0
    cases = []
    for i in range(10_000):
        c = CC.random_case(rng, i, dids)
        if check(vcc, c, d) is None:
            host += 1
        else:
            built += 1
        if i < 200:
            cases.append(c)
    assert built > 2000 and host > 1000
    total = sum(bound([c]) for c in cases)
    assert bound(cases) == total                                   # additive over workflows
    assert bound(cases[:0]) == 0


def test_time_text(vcc):
    out = np.zeros(64, dtype=np.uint8)
    for sec in (0, -1, 86399, CC.T0, -62135596800, 253402300799):
        for nsec in (0, 1, 10, 500_000_000, 999_999_999, 120_000_000):
            for zone in (0, 60, -60, 19800, -28800, 86340, -86340, 30, 86400, -86400):
                n = vcc.hs_vcc_time(C.c_int64(sec), C.c_int64(nsec), C.c_int64(zone), P(out))
                if not CO.time_ok(sec, nsec, zone):
                    assert n == 0
                    continue
                assert out[:n].tobytes() == CO.marshal_time(sec, nsec, zone), (sec, nsec, zone)


def test_did_filter(vcc):
    wanted = lambda d: bool(vcc.hs_vcc_did_wanted(d, len(d)))
    for d in (b"", b"did:key:", b" ", b"\t\n\v\f\r", "　".encode(), "\u0085        ".encode()):
        assert not wanted(d) and (d in (b"", b"did:key:") or CO.is_space_only(d))
    for d in (b"did:key:x", b"did:", b"did:key: ", b"\xff", b"\xe3\x80", "​".encode(), b"\x1c", b" x "):
        assert wanted(d) and not (d in (b"", b"did:key:") or CO.is_space_only(d))


def test_device_call_bound_equals_the_library_bound():
    """ExpandedKeys._chain_bound_dev (what workflow_chain_dev sizes its output with, from the offset arrays' ends alone) equals
    afc_vc_workflow_chain_bound on the same arrays, for whole batches and for batches that start past record 0."""
    import torch
    from agentfield_b200 import _abi
    from agentfield_b200.identity import ExpandedKeys
    lib = _abi.load()
    rng = np.random.default_rng(78)
    dids = CC.random_dids()
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x).view(np.int64))
    for trial in range(20):
        cases = [CC.random_case(rng, i, dids) for i in range(int(rng.integers(1, 40)))]
        a = CC.pack(cases)
        n = len(cases)
        i0 = int(rng.integers(0, n))
        k = n - i0
        arrays = (a[1][7 * i0:], a[2][i0:], a[4], a[7][2 * i0:], a[10])
        want = lib.afc_vc_workflow_chain_bound(*[_abi.ptr(np.ascontiguousarray(x)) for x in arrays], k)
        assert ExpandedKeys._chain_bound_dev(k, *[t(x) for x in arrays]) == want > 0
