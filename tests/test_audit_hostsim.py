"""The audit logic of the stored-document parser (agentfield_b200/csrc/afc_vcdoc.cuh: the capturing walk of k_vc_parse_capture and the
cross-check of k_vc_crosscheck), compiled for the CPU (tests/hostsim/hostsim_audit.cpp), against the host mirror's checks
(services.VCService._audit_component, _is_rfc3339, normalize_execution_status): column equality on the golden and random issued
documents against every class of column value, the status rule over all names, a timestamp corpus, and @context / type lists."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from agentfield_b200 import _abi, go_json as GJ
from agentfield_b200.services import _is_rfc3339, normalize_execution_status, _STATUS_ALIASES, _STATUS_CANONICAL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXEC, WF = 0, 1
UNDECIDED = 255
STATUS_IDS = {"unknown": 0, "pending": 1, "queued": 2, "running": 3, "succeeded": 4, "failed": 5, "cancelled": 6, "timeout": 7}
COLS = _abi.AUDIT_COLUMNS
STATUS_BIT = 1 << COLS.index("status")


@pytest.fixture(scope="module")
def audsim(tmp_path_factory):
    """TEST-ONLY CPU build of the audit logic (tests/hostsim/hostsim_audit.cpp), compiled into a temporary directory."""
    out = str(tmp_path_factory.mktemp("audsim") / "libafc_audsim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_audit.cpp")])
    lib = C.CDLL(out)
    lib.hs_audit_mask.restype = C.c_uint32
    lib.hs_status_class.restype = C.c_uint32
    lib.hs_rfc3339.restype = C.c_uint32
    lib.hs_status_class.argtypes = [C.c_char_p, C.c_uint64, C.c_int]
    lib.hs_rfc3339.argtypes = [C.c_char_p, C.c_uint32]
    return lib


def span_of(s):
    """The body of a string as json.Marshal writes it (what the parser records as the member's span)."""
    return GJ.string(s)[1:-1].encode("utf-8")


def capture(lib, kind, doc):
    cap = (C.c_uint32 * lib.hs_cap_words())()
    ok = lib.hs_audit_capture(kind, doc, C.c_uint64(len(doc)), cap)
    assert ok in (0, 1)
    return cap if ok else None


def device_mask(lib, kind, doc, cap, row=None):
    if row is None:
        return lib.hs_audit_mask(kind, doc, cap, None, None)
    flat = [v.encode("utf-8", "surrogatepass") if isinstance(v, str) else v for v in row]
    off = np.zeros(len(flat) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(v) for v in flat])
    buf = b"".join(flat) + b"\0"
    return lib.hs_audit_mask(kind, doc, cap, buf, off.ctypes.data_as(C.POINTER(C.c_uint64)))


def _decided_status_bytes(b, is_span):
    if is_span:
        return all(0x20 <= c <= 0x7E and c != 0x5C for c in b)
    return all(0x20 <= c <= 0x7E or 0x09 <= c <= 0x0D for c in b)


def mirror_mask(kind, doc_bytes, row=None):
    """The bits the device must report, from the strictly parsed document and the mirror's own rules (undecided where the device
    is told to leave a rule to the host)."""
    d = json.loads(doc_bytes)
    tl = d.get("type") or []
    if kind == WF:
        return 0 if {"VerifiableCredential", "AgentFieldWorkflowCredential"} <= set(tl) else _abi.AUDIT_NOT_AGENTFIELD
    cs, ex = d["credentialSubject"], d["credentialSubject"]["execution"]
    vals = [d["issuer"], cs["executionId"], cs["workflowId"], cs["sessionId"], cs["caller"]["did"], cs["target"]["did"], ex["status"],
            ex["inputHash"], ex["outputHash"], d["proof"]["proofValue"]]
    m = 0
    for k, (col, val) in enumerate(zip(row, vals)):
        cb = col.encode("utf-8", "surrogatepass") if isinstance(col, str) else col
        if k == COLS.index("status"):
            span = span_of(val)
            if not (_decided_status_bytes(span, True) and _decided_status_bytes(cb, False)):
                m |= _abi.AUDIT_STATUS_UNDECIDED
            elif normalize_execution_status(cb.decode()) != normalize_execution_status(val):
                m |= 1 << k
        elif cb != val.encode("utf-8"):
            m |= 1 << k
    date_span = span_of(d["issuanceDate"])
    if any(c >= 0x80 for c in date_span):
        m |= _abi.AUDIT_TIMESTAMP_UNDECIDED
    elif not _is_rfc3339(d["issuanceDate"]):
        m |= _abi.AUDIT_INVALID_TIMESTAMP
    for name, bit in (("@context", _abi.AUDIT_MISSING_CONTEXT), ("type", _abi.AUDIT_MISSING_TYPE), ("id", _abi.AUDIT_MISSING_ID),
                      ("issuer", _abi.AUDIT_MISSING_ISSUER), ("issuanceDate", _abi.AUDIT_MISSING_ISSUANCE_DATE)):
        if not d.get(name):
            m |= bit
    if "https://www.w3.org/2018/credentials/v1" not in (d.get("@context") or []):
        m |= _abi.AUDIT_NOT_W3C
    if not {"VerifiableCredential", "AgentFieldExecutionCredential"} <= set(tl):
        m |= _abi.AUDIT_NOT_AGENTFIELD
    return m


def record_row(doc_bytes):
    d = json.loads(doc_bytes)
    cs, ex = d["credentialSubject"], d["credentialSubject"]["execution"]
    return [d["issuer"], cs["executionId"], cs["workflowId"], cs["sessionId"], cs["caller"]["did"], cs["target"]["did"], ex["status"],
            ex["inputHash"], ex["outputHash"], d["proof"]["proofValue"]]


def column_variants(v):
    """Every class of column value against a document member v: equal, one byte off, prefix / suffix, empty, values that need
    escaping, invalid UTF-8."""
    b = v.encode("utf-8")
    out = [v, "", v + "x", "x" + v, v + '"', v + "\\", "<>&" + v, v + "\x01", v + " ", v + " ", b + b"\xff", b"\xc3" + b,
           b + b"\xed\xa0\x80", v + "�"]
    if b:
        out += [b[:-1], b[1:], bytes([b[0] ^ 1]) + b[1:], b[:-1] + bytes([b[-1] ^ 0x20])]
    return out


def _random_exec_docs(n, seed):
    from test_vcdoc_hostsim import _rand_exec
    rng = np.random.default_rng(seed)
    return [_rand_exec(rng, rng.integers(0, 256, 64, dtype=np.uint8).tobytes())[1] for _ in range(n)]


def _check_doc(lib, doc, rows):
    cap = capture(lib, EXEC, doc)
    if cap is None:
        from test_vcdoc_hostsim import _FLOATISH, _metadata
        assert b"\\ufffd" in doc or _FLOATISH.search(_metadata(doc)), doc[:200]      # the parser's only declines for what the issue path writes
        return 0
    for row in rows:
        assert device_mask(lib, EXEC, doc, cap, row) == mirror_mask(EXEC, doc, row), (row, doc[:300])
    return 1


def test_column_equality_golden_and_random(audsim):
    """Every column against every class of value, on the golden documents and 600 random issued ones: the device's bit is set
    exactly when the mirror's comparison fails (and the whole mask equals the mirror's)."""
    from test_vcdoc_hostsim import _golden_docs
    docs = [d for k, d, _ in _golden_docs() if k == EXEC] + _random_exec_docs(600, 0xA0D1)
    checked = 0
    for doc in docs:
        try:
            json.loads(doc)
        except ValueError:
            continue
        base = record_row(doc)
        rows = [base]
        for k in range(len(COLS)):
            for v in column_variants(base[k]):
                rows.append(base[:k] + [v] + base[k + 1:])
        checked += _check_doc(audsim, doc, rows)
    assert checked > 500


def test_golden_and_issued_documents_are_clean_against_their_records(audsim):
    """A document the issue path writes, against the record written with it, reports nothing but what its own values deserve."""
    from test_vcdoc_hostsim import _golden_docs
    for kind, doc, _ in _golden_docs():
        cap = capture(audsim, kind, doc)
        if cap is None:
            continue
        row = record_row(doc) if kind == EXEC else None
        m = device_mask(audsim, kind, doc, cap, row)
        assert m == mirror_mask(kind, doc, row)
        if kind == EXEC:
            assert m & ((1 << len(COLS)) - 1) == 0


def _case_variants(name):
    return {name, name.upper(), name.title(), name.capitalize(), "".join(c.upper() if i % 2 else c for i, c in enumerate(name)),
            "".join(c if i % 2 else c.upper() for i, c in enumerate(name))}


WS = ["", " ", "\t", "\n", "\v", "\f", "\r", "  \t\r\n"]


def test_status_rule(audsim):
    """All 24 names (8 canonical, 16 aliases) in every case and whitespace variant, in a column and in a document span: the device's
    class is the mirror's normalised name; the non-ASCII and U+001C-U+001F inputs are undecided."""
    names = sorted(_STATUS_CANONICAL) + sorted(_STATUS_ALIASES)
    assert len(names) == 24
    n_decided = 0
    for name in names + ["", "bogus", "succeeded!", "in progress", "x" * 40]:
        for v in _case_variants(name):
            for a in WS:
                for b in WS:
                    s = a + v + b
                    want = STATUS_IDS[normalize_execution_status(s)]
                    raw = s.encode()
                    assert audsim.hs_status_class(raw, len(raw), 0) == want, repr(s)
                    span = span_of(s)
                    got = audsim.hs_status_class(span, len(span), 1)
                    assert got == (want if b"\\" not in span else UNDECIDED), repr(s)
                    n_decided += got != UNDECIDED
    assert n_decided > 500
    for s in ["\x1csucceeded", "succeeded\x1f", "oK", "ſuccess", "succeeded ", "\u0085done", "café", "succeeded\x7f",
              "\x00ok", "ok\x1b"]:
        raw = s.encode()
        assert audsim.hs_status_class(raw, len(raw), 0) == UNDECIDED, repr(s)
        span = span_of(s)
        assert audsim.hs_status_class(span, len(span), 1) == UNDECIDED, repr(s)


def _timestamp_corpus():
    good = "2024-02-29T23:59:59Z"
    out = [good, "2026-09-21T06:00:00Z", "2026-09-21T06:00:00.5Z", "2026-09-21T06:00:00.123456789Z", "2026-09-21T06:00:00+05:30",
           "2026-09-21T06:00:00-23:59", "2026-09-21T06:00:00.1-00:00", "2026-09-21t06:00:00Z", "2026-09-21T06:00:00z", "2026-09-21 06:00:00Z",
           "2026-09-21T06:00:00", "2026-09-21T06:00Z", "2026-09-21", "2026-09-21T06:00:00.Z", "2026-09-21T06:00:00+0530", "2026-09-21T06:00:00+05",
           "2026-09-21T06:00:00+24:00", "2026-09-21T06:00:00+23:60", "2026-09-21T06:00:00ZZ", "2026-09-21T06:00:00Z ", " 2026-09-21T06:00:00Z",
           "2026-9-21T06:00:00Z", "26-09-21T06:00:00Z", "+2026-09-21T06:00:00Z", "", "Z", "2026-09-21T06:00:00.+01:00", "2026-09-21T06:00:00,5Z",
           "2026-09-21T06:00:00\n", "2026-09-21T06:00:00Z\n", "2026-09-21T06:00:00<Z", "\"2026-09-21T06:00:00Z", "2026-09-21T06:00:00\\Z",
           "2026-09-21T06:00:00 ", "2026-09-21T06:00:00.١Z", "٢٠٢٦-09-21T06:00:00Z", "2026-09-21T06:00:00é"]
    for y in ("0000", "1900", "2000", "2023", "2024", "9999", "0001", "2100", "2400"):
        for md in ("02-28", "02-29", "02-30", "01-31", "01-32", "04-30", "04-31", "06-31", "09-31", "11-31", "12-31", "13-01", "00-10", "05-00"):
            out.append("%s-%sT12:00:00Z" % (y, md))
    for h in ("00", "23", "24", "99"):
        for mi in ("00", "59", "60"):
            for sec in ("00", "59", "60", "61"):
                out.append("2026-09-21T%s:%s:%sZ" % (h, mi, sec))
    for i in range(len(good)):
        out.append(good[:i] + good[i + 1:])
        out.append(good[:i] + "x" + good[i + 1:])
        out.append(good[:i] + "0" + good[i + 1:])
    return out


def test_timestamp_rule(audsim):
    """A corpus against _is_rfc3339: every field at its boundaries, leap days in 0000 / 1900 / 2000 / 2023 / 2024, fractions, Z and
    offsets, lower-case t and z, missing parts, escapes; Arabic-Indic digits (and other non-ASCII text) are undecided."""
    valid = 0
    for ts in _timestamp_corpus():
        span = span_of(ts)
        got = audsim.hs_rfc3339(span, len(span))
        if any(c >= 0x80 for c in span):
            assert got == UNDECIDED, repr(ts)
        else:
            assert got == (0 if _is_rfc3339(ts) else 1), repr(ts)
            valid += got == 0
    assert valid > 50
    for ts, want in (("0000-02-29T00:00:00Z", 0), ("1900-02-29T00:00:00Z", 1), ("2000-02-29T00:00:00Z", 0), ("2023-02-29T00:00:00Z", 1),
                     ("2024-02-29T00:00:00Z", 0)):
        assert audsim.hs_rfc3339(ts.encode(), len(ts)) == want and _is_rfc3339(ts) == (want == 0), ts


W3C = "https://www.w3.org/2018/credentials/v1"


def _exec_doc(context, types, **cs):
    from test_vcdoc_hostsim import _proof
    doc = {"@context": context, "type": types, "id": "urn:agentfield:vc:1", "issuer": "did:key:z6Mk1", "issuanceDate": "2026-09-21T06:00:00Z",
           "credentialSubject": {"executionId": "e", "workflowId": "w", "sessionId": "s", "caller": {"did": "did:key:z6Mk1", "type": "agent", "agentNodeDid": "n"},
                                 "target": {"did": "t", "agentNodeDid": "n", "functionName": "f"},
                                 "execution": {"inputHash": "i", "outputHash": "o", "timestamp": "2026-09-21T06:00:00Z", "durationMs": 5,
                                               "status": "succeeded", "errorMessage": ""},
                                 "audit": {"inputDataHash": "", "outputDataHash": "", "metadata": None}}}
    for k, v in cs.items():
        doc[k] = v
    return GJ.vc_document(doc, _proof(doc["issuer"], bytes(64)))


def test_context_and_type_lists(audsim):
    """@context / type null, empty, without the literal, with the literal next to an escaped character, with duplicates; a literal
    written with an escape Go never uses leaves the document to the host."""
    types_ok = ["VerifiableCredential", "AgentFieldExecutionCredential"]
    cases = [(None, types_ok), ([], types_ok), ([W3C], None), ([W3C], []), ([W3C + "\n"], types_ok), (["<" + W3C], types_ok), ([W3C, W3C], types_ok),
             (["x", W3C], ["AgentFieldExecutionCredential"]), ([W3C], ["VerifiableCredential"]), ([W3C], ["VerifiableCredential", "AgentFieldWorkflowCredential"]),
             ([W3C], ["AgentFieldExecutionCredential", "x", "VerifiableCredential"]), ([W3C.upper()], ["verifiablecredential", "AgentFieldExecutionCredential"]),
             ([W3C[:-1]], ["VerifiableCredential ", "AgentFieldExecutionCredential"]), ([""], [""]), ([W3C], types_ok)]
    for context, types in cases:
        doc = _exec_doc(context, types)
        cap = capture(audsim, EXEC, doc)
        assert cap is not None, doc[:200]
        row = record_row(doc)
        assert device_mask(audsim, EXEC, doc, cap, row) == mirror_mask(EXEC, doc, row), (context, types)
    for extra in ({"id": ""}, {"issuer": ""}, {"issuanceDate": ""}, {"issuanceDate": "2026-02-30T00:00:00Z"}):
        doc = _exec_doc([W3C], types_ok, **extra)
        cap = capture(audsim, EXEC, doc)
        row = record_row(doc)
        m = device_mask(audsim, EXEC, doc, cap, row)
        assert m == mirror_mask(EXEC, doc, row) and m != 0, extra
    escaped = _exec_doc([W3C], types_ok).replace(b"https://www.w3.org", b"https:\\/\\/www.w3.org", 1)
    assert capture(audsim, EXEC, escaped) is None
    # workflow documents: only the AgentField type rule
    from test_vcdoc_hostsim import _rand_wf
    rng = np.random.default_rng(0xA0D2)
    n = 0
    for i in range(100):
        d, raw = _rand_wf(rng, bytes(64))
        if i % 3 == 0:
            d["type"] = ["VerifiableCredential", "AgentFieldWorkflowCredential"] if i % 2 else ["AgentFieldWorkflowCredential"]
            from test_vcdoc_hostsim import _proof
            raw = GJ.workflow_vc_document(d, _proof(d["issuer"], bytes(64)))
        cap = capture(audsim, WF, raw)
        if cap is None:
            continue
        assert device_mask(audsim, WF, raw, cap) == mirror_mask(WF, raw)
        n += 1
    assert n > 50
