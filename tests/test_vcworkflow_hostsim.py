"""The workflow-credential routines (agentfield_b200/csrc/afc_vcworkflow.cuh), compiled for the CPU (tests/hostsim/hostsim_vcworkflow.cpp),
against the oracle: the signing message and stored document of generateWorkflowVCDocument (oracle/ref_vc.py) for 0, 1 and many records
and strings of every escape class and invalid UTF-8; determineWorkflowStatus over all 24 status spellings and random multisets; the
records that send a workflow to the host; the RFC 3339 text against datetime; the first-record rule on ties.  Also checks that the sizes
pass and the fill pass agree and that afc_vc_workflow_bound (libafcrypto.so, host arithmetic only) is at least the real size."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import workflow_cases as WC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = 0xFE                 # never in a document: json.Marshal writes a 0xFE byte as �


@pytest.fixture(scope="module")
def vcw(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("vcwsim") / "libafc_vcwsim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_vcworkflow.cpp")])
    return C.CDLL(out)


def run(vcw, case, fill=True):
    """(summary, state, message, document) as the kernels write them for one workflow; the byte strings are None for a HOST workflow.
    The buffers start as SENTINEL bytes: the fill and id passes must write exactly the lengths the sizes pass reported."""
    cols, coff, _, rcols, rcoff, created = WC.pack([case])
    created = np.ascontiguousarray(created if len(created) else np.zeros(2, dtype=np.int64))
    summ, state = (C.c_uint32 * 4)(), C.c_uint32()
    ml, dl = C.c_uint64(), C.c_uint64()
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    args = (P(cols), P(coff), P(rcols), P(rcoff), P(created), len(case["records"]), summ, C.byref(state))
    assert vcw.hs_vcw_issue(*args, None, C.byref(ml), None, C.byref(dl)) == 0
    if state.value == 1 or not fill:
        return list(summ), state.value, None, None
    msg = np.full(ml.value + 32, SENTINEL, dtype=np.uint8)
    doc = np.full(dl.value + 32, SENTINEL, dtype=np.uint8)
    ml2, dl2 = C.c_uint64(), C.c_uint64()
    assert vcw.hs_vcw_issue(*args, P(msg), C.byref(ml2), P(doc), C.byref(dl2)) == 0
    assert (ml2.value, dl2.value) == (ml.value, dl.value)
    for buf, n in ((msg, ml.value), (doc, dl.value)):
        assert not (buf[:n] == SENTINEL).any(), "a byte the sizes pass counted was not written"
        assert (buf[n:] == SENTINEL).all(), "a byte past the counted length was written"
    return list(summ), state.value, msg[:ml.value].tobytes(), doc[:dl.value].tobytes()


def check(vcw, case):
    summ, state, msg, doc = run(vcw, case)
    want = WC.summary(case)
    if want is None:
        assert state == 1 and summ == [0, 0, 0, 0] and msg is None
        return
    assert state == 0 and summ == want, (summ, want)
    wmsg, wdoc = WC.oracle_docs(case)
    assert msg == wmsg
    assert doc == wdoc


def test_zero_one_and_many_records(vcw):
    check(vcw, {"cols": WC.base_cols(), "records": []})
    check(vcw, {"cols": WC.base_cols(), "records": [(b"vc-1790000000000000001", b"succeeded", 1_790_000_000, 5)]})
    check(vcw, {"cols": WC.base_cols(), "records": [(b"vc-1", b"running", 1_790_000_000, 5)]})
    many = [(b"vc-%d" % (1_790_000_000_000_000_000 + j), b"completed", 1_790_000_000 + j % 97, (j * 7919) % 10 ** 9) for j in range(3000)]
    check(vcw, {"cols": WC.base_cols(), "records": many})


def test_escape_classes_and_invalid_utf8(vcw):
    for k in range(7):
        for odd in WC.ODD:
            cols = WC.base_cols()
            cols[k] = cols[k] + odd
            check(vcw, {"cols": cols, "records": [(b"vc-1" + odd, b"done", 1_790_000_000, 0), (odd, b"failed", 1_790_000_001, 0)]})
            check(vcw, {"cols": cols, "records": []})
    rng = np.random.default_rng(41)
    for i in range(400):
        check(vcw, WC.random_case(rng, i, WC.base_cols()[2], odd=0.3))


def test_all_status_spellings(vcw):
    for sp in WC.STATUS_SPELLINGS:
        for v in (sp, sp.upper(), sp.title(), " " + sp, sp + "\t", "\n\v" + sp.upper() + " \f\r", "x" + sp, sp + "x", sp.replace("_", " ")):
            case = {"cols": WC.base_cols(), "records": [(b"vc-1", v.encode(), 1_790_000_000, 0)]}
            summ, state, _, _ = run(vcw, case, fill=False)
            assert state == 0 and summ == WC.summary(case), (v, summ)
            check(vcw, case)
    for v in ("", " ", "\t\n", "succeeded!", "a" * 12, "processing1"):
        assert run(vcw, {"cols": WC.base_cols(), "records": [(b"vc-1", v.encode(), 1_790_000_000, 0)]}, fill=False)[0][0] == 0


def test_random_multisets(vcw):
    rng = np.random.default_rng(42)
    seen = set()
    for i in range(3000):
        case = WC.random_case(rng, i, WC.base_cols()[2], max_records=int(rng.choice([3, 8, 40])))
        summ, state, _, _ = run(vcw, case, fill=False)
        assert state == 0 and summ == WC.summary(case), i
        seen.add(summ[0])
        if i % 10 == 0:
            check(vcw, case)
    assert seen == set(range(8))


def test_undecided_statuses_go_to_the_host(vcw):
    for b in list(range(0, 9)) + list(range(0x0E, 0x20)) + [0x7F, 0x80, 0xC3, 0xE2, 0xFF]:
        st = b"succ" + bytes([b]) + b"eeded"
        case = {"cols": WC.base_cols(), "records": [(b"vc-1", b"succeeded", 1_790_000_000, 0), (b"vc-2", st, 1_790_000_001, 0)]}
        assert WC.is_host(case)
        check(vcw, case)
    check(vcw, {"cols": WC.base_cols(), "records": [(b"vc-1", "\u212aelvin".encode(), 1_790_000_000, 0)]})      # Kelvin sign: ToLower is Unicode
    check(vcw, {"cols": WC.base_cols(), "records": [(b"vc-1", "done\u00a0".encode(), 1_790_000_000, 0)]})       # NBSP: TrimSpace is Unicode


def test_time_text_against_datetime(vcw):
    import datetime as dt
    e = dt.datetime(1970, 1, 1)
    named = [0, -1, 1, 86399, 86400, -86400, -86401, int((dt.datetime(2000, 2, 29, 12, 34, 56) - e).total_seconds()),
             int((dt.datetime(1900, 3, 1) - e).total_seconds()), int((dt.datetime(1900, 2, 28, 23, 59, 59) - e).total_seconds()),
             int((dt.datetime(2100, 3, 1) - e).total_seconds()), int((dt.datetime(1600, 2, 29) - e).total_seconds()), WC.SEC_MIN, WC.SEC_MAX,
             WC.SEC_MIN + 1, WC.SEC_MAX - 1]
    rng = np.random.default_rng(43)
    secs = np.array(named + list(rng.integers(WC.SEC_MIN, WC.SEC_MAX + 1, 100_000)), dtype=np.int64)
    out = np.zeros(20 * len(secs), dtype=np.uint8)
    vcw.hs_vcw_times(secs.ctypes.data_as(C.c_void_p), len(secs), out.ctypes.data_as(C.c_void_p))
    got = out.tobytes()
    for i, s in enumerate(secs.tolist()):
        assert got[20 * i:20 * i + 20].decode() == WC.time_text(s), s
    assert WC.time_text(WC.SEC_MIN) == "0001-01-01T00:00:00Z" and WC.time_text(WC.SEC_MAX) == "9999-12-31T23:59:59Z"
    assert WC.time_text(0) == "1970-01-01T00:00:00Z"


def test_time_range_and_nanoseconds(vcw):
    st = b"succeeded"
    cls = lambda s, ns: vcw.hs_vcw_record_class(st, len(st), C.c_int64(s), C.c_int64(ns))
    assert cls(WC.SEC_MIN, 0) == 4 and cls(WC.SEC_MAX, 999_999_999) == 4
    assert cls(WC.SEC_MIN - 1, 999_999_999) == 8 and cls(WC.SEC_MAX + 1, 0) == 8
    assert cls(0, -1) == 8 and cls(0, 10 ** 9) == 8 and cls(-(2 ** 63), 0) == 8 and cls(2 ** 63 - 1, 0) == 8
    for s, ns in ((WC.SEC_MIN, 0), (WC.SEC_MAX, 999_999_999), (-1, 999_999_999), (0, 0)):
        check(vcw, {"cols": WC.base_cols(), "records": [(b"vc-1", st, s, ns), (b"vc-2", b"failed", 1_790_000_000, 1)]})
    for s, ns in ((WC.SEC_MIN - 1, 0), (WC.SEC_MAX + 1, 0), (0, 10 ** 9), (0, -1)):
        check(vcw, {"cols": WC.base_cols(), "records": [(b"vc-1", st, s, ns), (b"vc-2", b"failed", 1_790_000_000, 1)]})


def test_ties_pick_the_first_record(vcw):
    t = 1_790_000_000
    recs = [(b"vc-a", b"done", t + 5, 7), (b"vc-b", b"done", t, 3), (b"vc-c", b"done", t, 3), (b"vc-d", b"done", t + 5, 7), (b"vc-e", b"ok", t, 2)]
    summ, _, _, _ = run(vcw, {"cols": WC.base_cols(), "records": recs[:4]})
    assert summ[2:] == [1, 0]
    summ, _, _, _ = run(vcw, {"cols": WC.base_cols(), "records": recs})
    assert summ[2:] == [4, 0]
    same = [(b"vc-%d" % j, b"failed", t, 999_999_999) for j in range(6)]
    assert run(vcw, {"cols": WC.base_cols(), "records": same})[0] == [5, 0, 0, 0]
    check(vcw, {"cols": WC.base_cols(), "records": recs})


def test_bound_covers_escape_heavy_inputs(vcw):
    from agentfield_b200 import _abi
    lib = _abi.load()
    heavy = [b"\x01" * 64, b"\xff" * 64, b"<>&" * 20, "\u2028".encode() * 20, b'"\\' * 32]
    cases = []
    for h in heavy:
        cases.append({"cols": [h] * 7, "records": [(h, b"done", 1_790_000_000, 0)] * 9})
        cases.append({"cols": [h] * 7, "records": []})
        cases.append({"cols": WC.base_cols(), "records": [(b"", b"failed", 0, 0)] * 50})
    total = 0
    for c in cases:
        _, _, msg, doc = run(vcw, c)
        cols, coff, roff, rcols, rcoff, _ = WC.pack([c])
        bound = lib.afc_vc_workflow_bound(_abi.ptr(coff), _abi.ptr(roff), _abi.ptr(rcoff), 1)
        assert bound >= len(doc) and bound >= len(msg)
        total += len(doc)
    cols, coff, roff, rcols, rcoff, _ = WC.pack(cases)
    assert lib.afc_vc_workflow_bound(_abi.ptr(coff), _abi.ptr(roff), _abi.ptr(rcoff), len(cases)) >= total
    assert lib.afc_vc_workflow_bound(_abi.ptr(coff), _abi.ptr(roff), _abi.ptr(rcoff), 0) == 0
