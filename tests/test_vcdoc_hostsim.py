"""The stored-document parser (agentfield_b200/csrc/afc_vcdoc.cuh), compiled for the CPU (tests/hostsim/hostsim_vcdoc.cpp), against the host mirror of
what the reference verifies: for every document it either declines (HOST), or the document parses strictly, the signing bytes it
builds equal go_json's re-marshalling with a zero proof, the signature it decodes equals the base64url decode of proofValue and the
issuer span is the parsed issuer.  Inputs: the golden Go cases, random issued documents, every single-byte mutation of a few of
them and targeted non-canonical rewrites; coverage checks show it does not simply decline everything."""
import base64
import ctypes as C
import json
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import golden
from agentfield_b200 import go_json as GJ

HOST, VALID, INVALID, BAD_ENCODING = 2, 1, 0, 4
EXEC, WF = 0, 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def vcsim(tmp_path_factory):
    """TEST-ONLY CPU build of afc_vcdoc.cuh (tests/hostsim/hostsim_vcdoc.cpp), compiled into a temporary directory."""
    out = str(tmp_path_factory.mktemp("vcsim") / "libafc_vcsim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_vcdoc.cpp")])
    return C.CDLL(out)


def run(vcsim, kind, doc):
    msg = (C.c_uint8 * (len(doc) + 64))()
    ml, sig, sp = C.c_uint64(), (C.c_uint8 * 64)(), (C.c_uint32 * 5)()
    st = vcsim.hs_vc_parse(kind, doc, C.c_uint64(len(doc)), msg, C.byref(ml), sig, sp)
    assert st in (0, 1, 2, 4), st
    return st, bytes(msg)[:ml.value], bytes(sig), list(sp)


# ---- strict parse: what the reference's Unmarshal yields for a document that has exactly the struct's members
_S, _L, _I, _P, _M = "s", "l", "i", "p", "m"
_CALLER = {"did": _S, "type": _S, "agentNodeDid": _S}
_AUDIT = {"inputDataHash": _S, "outputDataHash": _S, "metadata": _M}
_PROOF = {"type": _S, "created": _S, "verificationMethod": _S, "proofPurpose": _S, "proofValue": _S}
SCHEMA = {
    EXEC: {"@context": _L, "type": _L, "id": _S, "issuer": _S, "issuanceDate": _S,
           "credentialSubject": {"executionId": _S, "workflowId": _S, "sessionId": _S, "caller": _CALLER,
                                 "target": {"did": _S, "agentNodeDid": _S, "functionName": _S},
                                 "execution": {"inputHash": _S, "outputHash": _S, "timestamp": _S, "durationMs": _I, "status": _S, "errorMessage": _S},
                                 "audit": _AUDIT}, "proof": _PROOF},
    WF: {"@context": _L, "type": _L, "id": _S, "issuer": _S, "issuanceDate": _S,
         "credentialSubject": {"workflowId": _S, "sessionId": _S, "componentVcIds": _L, "totalSteps": _I, "completedSteps": _I, "status": _S,
                               "startTime": _S, "endTime": _P, "snapshotTime": _S, "orchestrator": _CALLER, "audit": _AUDIT},
         "proof": _PROOF}}
OPTIONAL = {"errorMessage", "endTime"}


class Strict(Exception):
    pass


def strict_parse(doc, kind):
    class O(list):
        pass
    try:
        # "-0" stays a (negative zero) float as in Go's interface{} decoding; in an int member it then fails the type check
        v = json.loads(doc.decode("utf-8"), object_pairs_hook=lambda ps: O(tuple(p) for p in ps), parse_int=lambda t: -0.0 if t == "-0" else int(t))
    except (ValueError, UnicodeDecodeError) as ex:
        raise Strict(str(ex))

    def conv(x, t):
        if isinstance(t, dict):
            if not isinstance(x, O):
                raise Strict("not an object")
            keys = [k for k, _ in x]
            if len(set(keys)) != len(keys) or any(k not in t for k in keys) or any(k not in keys for k in t if k not in OPTIONAL):
                raise Strict("members")
            return {k: conv(y, t[k]) for k, y in x}
        if t in (_S, _P):
            if not isinstance(x, str) and not (t == _P and x is None):
                raise Strict("string")
            return x
        if t == _L:
            if x is not None and not (isinstance(x, list) and not isinstance(x, O) and all(isinstance(y, str) for y in x)):
                raise Strict("[]string")
            return x
        if t == _I:
            if isinstance(x, bool) or not isinstance(x, int):
                raise Strict("int")
            return x
        if x is not None and not isinstance(x, O):
            raise Strict("map")
        return iface(x)

    def iface(x):
        if isinstance(x, O):
            return {k: iface(y) for k, y in x}
        if isinstance(x, list):
            return [iface(y) for y in x]
        return GJ.unmarshal_numbers(x)
    d = conv(v, SCHEMA[kind])
    if kind == WF:
        d["credentialSubject"].setdefault("endTime", None)
    return d


def b64_status(pv):
    if not re.fullmatch(r"[A-Za-z0-9_-]*", pv) or len(pv) % 4 == 1:
        return BAD_ENCODING, None
    raw = base64.urlsafe_b64decode(pv + "=" * (-len(pv) % 4))
    return (VALID, raw) if len(raw) == 64 else (INVALID, None)


def check(vcsim, kind, doc):
    """Runs one document; asserts the parser's verdict is consistent with the strict parse; returns the status."""
    st, msg, sig, sp = run(vcsim, kind, doc)
    if st == HOST:
        return st
    try:
        d = strict_parse(doc, kind)
    except Strict as ex:
        raise AssertionError("accepted a document the strict parse rejects (%s): %r" % (ex, doc[:200]))
    want_st, raw = b64_status(d["proof"]["proofValue"])
    assert st == want_st, (st, want_st, d["proof"]["proofValue"])
    assert doc[sp[0]:sp[0] + sp[1]].decode() == d["issuer"]
    assert json.loads(b'"' + doc[sp[2]:sp[2] + sp[3]] + b'"') == d["issuanceDate"]
    if st == VALID:
        canon = GJ.vc_document(d) if kind == EXEC else GJ.workflow_vc_document(d)
        assert msg == canon, (msg[-200:], canon[-200:])
        assert sig == raw
    return st


def _golden_docs():
    g = golden("go_cases.json")
    return [(EXEC, c["expect_stored"].encode("utf-8"), c) for c in g["execution_vcs"]] + \
           [(WF, c["expect_stored"].encode("utf-8"), c) for c in g["workflow_vcs"]]


_FLOATISH = re.compile(rb'[:,\[]-?\d+(\.\d|[eE])|[:,\[]-?\d{16,}')


def _metadata(doc):
    return doc[doc.index(b'"metadata":'):doc.index(b',"proof":')]


def test_golden_documents(vcsim):
    """Every golden document is either verified on the device with exactly the reference's signing bytes and signature, or holds a
    metadata number the device leaves to the host (a fraction, an exponent or more than 15 digits) — and only then."""
    accepted = 0
    for kind, doc, c in _golden_docs():
        st, msg, sig, _ = run(vcsim, kind, doc)
        if _FLOATISH.search(_metadata(doc)) or b"\\ufffd" in doc:
            assert st == HOST, c["id"]
            continue
        assert st == VALID, c["id"]
        assert msg == c["expect_canonical"].encode("utf-8") and sig.hex() == c["expect_sig"]
        check(vcsim, kind, doc)
        accepted += 1
    assert accepted == 14           # the other six hold fractions or exponents in their metadata


_POOL = ["did:key:z6Mk", "urn:agentfield:vc:", "2026-09-21T06:00:00Z", "héllo", "日本語", "😀", "<a&b>", 'q"uote', "back\\slash", "tab\t",
         "nl\n", "\x01\x1f", "  ", "\x7f", "/", "", "plain text value", "�", "ü" * 7]


KEY_POOL = [p for p in _POOL if GJ.string(p)[1:-1] == p]


def _rand_str(rng, allow_bad=False):
    parts = [_POOL[i] for i in rng.integers(0, len(_POOL), rng.integers(0, 5))]
    if allow_bad and rng.random() < 0.004:
        parts.append("\ud800")                        # lone surrogate: Go writes �
    return "".join(parts)


def _rand_meta(rng, depth=0):
    r = rng.random()
    if depth == 0 and r < 0.15:
        return None
    # keys without characters Go escapes (an escaped key is left to the host); Go sorts them by bytes, as sorted() does here
    keys = sorted({"".join(KEY_POOL[j] for j in rng.integers(0, len(KEY_POOL), 2)) + str(k) for k in range(rng.integers(0, 5))})
    m = {}
    for k in keys:
        t = rng.integers(0, 8)
        if t == 0:
            m[k] = _rand_str(rng)
        elif t == 1:
            m[k] = float(int(rng.integers(-10**14, 10**14)))
        elif t == 2:
            m[k] = bool(rng.integers(0, 2))
        elif t == 3:
            m[k] = None
        elif t == 4 and depth < 3:
            m[k] = _rand_meta(rng, depth + 1) or {}
        elif t == 5 and depth < 3:
            m[k] = [_rand_str(rng), float(rng.integers(0, 100)), None, [], {}]
        elif t == 6:
            m[k] = -0.0
        else:
            m[k] = 0.0
    return m


def _rand_exec(rng, sig):
    s = lambda: _rand_str(rng, True)
    doc = {"@context": None if rng.random() < 0.1 else [s() for _ in range(rng.integers(0, 3))],
           "type": [] if rng.random() < 0.1 else ["VerifiableCredential", s()], "id": s(), "issuer": "did:key:z6Mk" + str(rng.integers(0, 99)),
           "issuanceDate": s(),
           "credentialSubject": {"executionId": s(), "workflowId": s(), "sessionId": s(), "caller": {"did": s(), "type": s(), "agentNodeDid": s()},
                                 "target": {"did": s(), "agentNodeDid": s(), "functionName": s()},
                                 "execution": {"inputHash": s(), "outputHash": s(), "timestamp": s(), "durationMs": int(rng.integers(-10**17, 10**17)),
                                               "status": s(), "errorMessage": s() if rng.random() < 0.5 else ""},
                                 "audit": {"inputDataHash": s(), "outputDataHash": s(), "metadata": _rand_meta(rng)}}}
    return doc, GJ.vc_document(doc, _proof(doc["issuer"], sig))


def _rand_wf(rng, sig):
    s = lambda: _rand_str(rng, True)
    end = None if rng.random() < 0.3 else ("" if rng.random() < 0.3 else s())
    doc = {"@context": [s()], "type": None if rng.random() < 0.2 else [s(), s()], "id": s(), "issuer": "did:key:z6Mk" + str(rng.integers(0, 99)),
           "issuanceDate": s(),
           "credentialSubject": {"workflowId": s(), "sessionId": s(), "componentVcIds": None if rng.random() < 0.2 else [s() for _ in range(rng.integers(0, 4))],
                                 "totalSteps": int(rng.integers(0, 1000)), "completedSteps": int(rng.integers(-5, 1000)), "status": s(), "startTime": s(),
                                 "endTime": end, "snapshotTime": s(), "orchestrator": {"did": s(), "type": s(), "agentNodeDid": s()},
                                 "audit": {"inputDataHash": s(), "outputDataHash": s(), "metadata": _rand_meta(rng)}}}
    return doc, GJ.workflow_vc_document(doc, _proof(doc["issuer"], sig))


def _proof(did, sig):
    return {"type": "Ed25519Signature2020", "created": "2026-09-21T06:00:00Z", "verificationMethod": did + "#key-1", "proofPurpose": "assertionMethod",
            "proofValue": base64.urlsafe_b64encode(sig).rstrip(b"=").decode()}


def test_random_issued_documents(vcsim):
    """Random documents as the issue path writes them (escapes, multibyte text, every metadata shape, both endTime forms): none is
    declined unless it holds \\ufffd (Go does not round-trip it), and every verdict is exact."""
    rng = np.random.default_rng(0xAFD0)
    n_dev = 0
    for i in range(600):
        sig = rng.integers(0, 256, 64, dtype=np.uint8).tobytes()
        kind = EXEC if i % 2 == 0 else WF
        _, doc = (_rand_exec if kind == EXEC else _rand_wf)(rng, sig)
        st = check(vcsim, kind, doc)
        if b"\\ufffd" in doc:
            assert st == HOST
        else:
            assert st == VALID, doc[:300]
            n_dev += 1
    assert n_dev > 400


SUBS = [b" ", b'"', b"\\", b"0", b"1", b"-", b".", b"e", b"A", b"{", b"}", b"[", b"]", b",", b"\x80", b"\xc3"]


def _mutation_sources():
    docs = [(k, d) for k, d, _ in _golden_docs()]
    pick = [docs[0], docs[1], docs[10], docs[13]]
    rng = np.random.default_rng(0xAFD1)
    sig = rng.integers(0, 256, 64, dtype=np.uint8).tobytes()
    while True:
        _, d = _rand_wf(rng, sig)
        if b"endTime" in d and b"\\ufffd" not in d and b"metadata\":{" in d:
            pick.append((WF, d))
            break
    return pick


@pytest.mark.parametrize("which", range(5))
def test_every_single_byte_mutation(vcsim, which):
    """Every single-byte deletion, duplication and substitution of a few documents: each verdict is exact, and swapping one plain
    character inside a string value for another is never declined."""
    kind, doc = _mutation_sources()[which]
    assert run(vcsim, kind, doc)[0] != HOST
    plain_at = _plain_string_bytes(doc)
    swaps = 0
    for i in range(len(doc)):
        for m in (doc[:i] + doc[i + 1:], doc[:i + 1] + doc[i:]):
            check(vcsim, kind, m)
        for b in SUBS:
            if doc[i:i + 1] == b:
                continue
            m = doc[:i] + b + doc[i + 1:]
            st = check(vcsim, kind, m)
            plain = lambda c: c.isalnum() and c.isascii()
            if i in plain_at and plain(b) and not _in_proof_value(doc, i):
                assert st != HOST, (i, b, doc[max(0, i - 20):i + 20])
                swaps += 1
    assert swaps > 100


def _plain_string_bytes(doc):
    """Positions of ASCII letters and digits inside JSON string VALUES (not member names), outside escape sequences."""
    out = set()
    for m in re.finditer(rb'":"((?:[^"\\]|\\.)*)"', doc):
        i = m.start(1)
        while i < m.end(1):
            if doc[i] == 0x5c:
                i += 6 if doc[i + 1] == 0x75 else 2
                continue
            if chr(doc[i]).isalnum() and doc[i] < 0x80:
                out.add(i)
            i += 1
    return out


def _in_proof_value(doc, i):
    k = doc.rfind(b'"proofValue":"')
    return k >= 0 and i >= k


def _rewrites(doc):
    """(rewritten document, True if it must go to the host, False if it must not, None if either is exact)"""
    s = doc.decode("utf-8")
    yield s.replace('","issuer"', '", "issuer"', 1), True
    yield s.replace('{"@context"', '{ "@context"', 1), True
    yield " " + s, True
    yield s + " ", True
    yield s + "\n", True
    yield s.replace('"id":', '"ID":', 1), True
    yield s.replace('"issuanceDate":"', '"issuanceDate":"x","issuanceDate":"', 1), True
    i, j = s.index('"id":'), s.index(',"issuer"')
    yield s[:i] + s[j + 1:s.index(',"issuanceDate"')] + "," + s[i:j] + s[s.index(',"issuanceDate"'):], True       # issuer before id
    yield s.replace('"metadata":{', '"metadata":{"zz":1,"aa":2,', 1), True
    yield s.replace('"metadata":{', '"metadata":{"a":1,"a":2,', 1), True
    # (number, must go to the host in metadata, ... in an int member)
    for num, in_meta, in_int in (("1.0", True, True), ("1e2", True, True), ("01", True, True), ("-0", False, True), ("1234567890123456", True, False),
                                 ("123456789012345", False, False), ("-123456789012345", False, False), ("0", False, False), ("1E2", True, True),
                                 ("+1", True, True)):
        yield s.replace('"metadata":{', '"metadata":{"!":%s,' % num, 1), in_meta
        yield re.sub(r'"(durationMs|totalSteps)":-?\d+', r'"\1":%s' % num, s, count=1), in_int
    yield re.sub(r'"(durationMs|totalSteps)":-?\d+', r'"\1":123456789012345678', s, count=1), False
    yield re.sub(r'"(durationMs|totalSteps)":-?\d+', r'"\1":1234567890123456789', s, count=1), True
    for esc, host in (("\\u0041", True), ("\\/", True), ("\\ufffd", True), ("\\ud83d\\ude00", True), ("\\u00e9", True), ("\\u003C", True),
                      ("\\u000a", True), ("\\u000b", False), ("\\u001f", False), ("\\u2028", False), ("\\u0026", False), ("\\t", False),
                      ("\\x", True), ("\\u007f", True)):
        yield s.replace('"id":"', '"id":"' + esc, 1), host
    yield s.replace('"id":"', '"id":"\u2028', 1), True                 # raw U+2028: Go escapes it
    yield s.replace('"id":"', '"id":"<', 1), True
    yield s.replace(',"type":[', ',"type":null,"x":[', 1), True
    yield re.sub(r'(,"status":"[^"]*")', r'\1,"errorMessage":""', s, count=1), True
    yield re.sub(r'(,"startTime":"[^"]*")', r'\1,"endTime":null', s, count=1), True
    yield re.sub(r'(,"startTime":"[^"]*")', r'\1,"endTime":""', s, count=1), None
    yield s.replace('"metadata":{', '"metadata":{"!":' + "[" * 9 + "]" * 9 + ",", 1), True      # deeper than the device follows
    yield s.replace('"metadata":{', '"metadata":{"!":' + "[" * 6 + "]" * 6 + ",", 1), False
    pv = re.search(r'"proofValue":"([^"]*)"', s).group(1)
    for new in (pv[:84], pv[:85], pv, pv + "A", pv[:-1] + "B", pv[:-1] + "_", pv[:10] + "+" + pv[11:], pv[:10] + "/" + pv[11:], pv + "==",
                pv[:10] + "é" + pv[12:], ""):
        yield s.replace('"proofValue":"%s"' % pv, '"proofValue":"%s"' % new), False
    yield s.replace('"proofValue":"%s"' % pv, '"proofValue":"%s"' % (pv[:10] + "\\n" + pv[10:])), True


def test_targeted_rewrites(vcsim):
    """Whitespace, re-ordered / re-cased / duplicated members, unsorted or duplicate metadata keys, non-integer numbers, -0, long
    integers, escapes Go never writes, surrogates, deep nesting, omitempty forms and malformed proofValues: exact verdicts, with
    the ones that must go to the host going there."""
    n = 0
    for kind, doc, _ in _golden_docs()[:2] + _golden_docs()[10:12]:
        for s, host in _rewrites(doc):
            raw = s.encode("utf-8", "surrogatepass")
            st = check(vcsim, kind, raw)
            if raw != doc and host is not None:
                assert (st == HOST) == host, (st, s[:160])
            n += 1
    assert n > 150
    # proofValue lengths: 84 / 87 characters decode to 63 / 65 bytes (INVALID), 85 is not base64 (BAD_ENCODING), non-zero trailing
    # bits are ignored as Go's default decoder does
    kind, doc, c = _golden_docs()[0]
    s = doc.decode()
    pv = re.search(r'"proofValue":"([^"]*)"', s).group(1)
    assert len(pv) == 86
    for new, want in ((pv[:84], INVALID), (pv[:85], BAD_ENCODING), (pv + "A", INVALID), (pv[:-1] + "_", VALID), (pv[:3] + "+" + pv[4:], BAD_ENCODING),
                      (pv[:3] + "=" + pv[4:], BAD_ENCODING), ("", INVALID)):
        raw = s.replace(pv, new).encode()
        assert run(vcsim, kind, raw)[0] == want, new
        check(vcsim, kind, raw)
