"""The tolerant document walk (agentfield_b200/csrc/afc_vcjson.cuh), compiled for the CPU (tests/hostsim/hostsim_vcjson.cpp), against the
host mirror of what the reference verifies: services.go_unmarshal_vc, then go_json's re-marshalling with the zero proof.  For every
input the walk either declines (HOST), or the mirror parses the document, the message the walk builds is byte for byte the mirror's,
the decoded signature is the base64url decode of proofValue, the status is the base64 status, and the issuer and issuanceDate
spans decode to the mirror's values.  Inputs: the golden Go cases in six client spellings, random issued documents re-spelled at
random, every single-byte mutation of two pretty-printed documents and targeted cases; coverage checks show it does not simply
decline everything."""
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
from agentfield_b200.respell import SPELLINGS, Num, parse_keep, spell, write  # noqa: F401 (also used by test_vcjson_gpu)
from agentfield_b200.services import go_unmarshal_vc
from test_vcdoc_hostsim import SUBS, _FLOATISH, _metadata, _rand_exec, _rand_wf

HOST, VALID, INVALID, BAD_ENCODING = 2, 1, 0, 4
EXEC, WF = 0, 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAIL = len(b'{"type":"","created":"","verificationMethod":"","proofPurpose":"","proofValue":""}}')


def build_cpu_walk(tmp_path_factory):
    """TEST-ONLY CPU build of afc_vcjson.cuh (tests/hostsim/hostsim_vcjson.cpp), compiled into a temporary directory."""
    out = str(tmp_path_factory.mktemp("vcjsim") / "libafc_vcjsim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_vcjson.cpp")])
    lib = C.CDLL(out)
    lib.hs_vcj_put_cp.restype = C.c_uint32
    lib.hs_go_json_escape.restype = C.c_uint64
    return lib


@pytest.fixture(scope="module")
def vcj(tmp_path_factory):
    return build_cpu_walk(tmp_path_factory)


def run(vcj, kind, doc):
    msg = (C.c_uint8 * (len(doc) + 64))()
    ml, sig, sp = C.c_uint64(), (C.c_uint8 * 64)(), (C.c_uint32 * 5)()
    st = vcj.hs_vcj_parse(kind, doc, C.c_uint64(len(doc)), msg, C.byref(ml), sig, sp)
    assert st in (0, 1, 2, 4), st
    return st, bytes(msg)[:ml.value], bytes(sig), list(sp)


def b64_status(pv):
    if not re.fullmatch(r"[A-Za-z0-9_-]*", pv) or len(pv) % 4 == 1:
        return BAD_ENCODING, None
    raw = base64.urlsafe_b64decode(pv + "=" * (-len(pv) % 4))
    return (VALID, raw) if len(raw) == 64 else (INVALID, None)


def mirror_message(d, kind):
    return GJ.vc_document(d) if kind == EXEC else GJ.workflow_vc_document(d)


def mirror_unmarshal(doc, kind):
    """services.go_unmarshal_vc, with a -0 in metadata kept as Go keeps it (a float64 negative zero, written back as -0).  The mirror
    reads integer tokens through int and writes 0 there; the device, like Go, writes -0.  The rest of the document is the mirror's."""
    d = go_unmarshal_vc(doc, kind)
    if re.search(rb"-0(?![.\deE])", doc):
        raw = json.loads(doc.decode("utf-8"), parse_int=lambda t: -0.0 if t == "-0" else int(t))
        d["credentialSubject"]["audit"]["metadata"] = GJ.unmarshal_numbers(raw["credentialSubject"]["audit"].get("metadata"))
    return d


def check(vcj, kind, doc):
    """Runs one document and asserts the invariant of the module docstring; returns (status, message)."""
    st, msg, sig, sp = run(vcj, kind, doc)
    if st == HOST:
        return st, None
    try:
        d = mirror_unmarshal(doc, kind)
    except ValueError as ex:
        raise AssertionError("accepted a document the mirror rejects (%s): %r" % (ex, doc[:200]))
    assert msg == mirror_message(d, kind), (msg[:300], mirror_message(d, kind)[:300], doc[:300])
    assert sp[4] + TAIL == len(msg) <= len(doc)
    want_st, raw = b64_status(d["proof"]["proofValue"])
    assert st == want_st, (st, want_st, d["proof"]["proofValue"])
    if st == VALID:
        assert sig == raw
    assert doc[sp[0]:sp[0] + sp[1]].decode() == d["issuer"]
    assert json.loads(b'"' + doc[sp[2]:sp[2] + sp[3]] + b'"') == d["issuanceDate"]
    return st, msg


def _golden_docs():
    g = golden("go_cases.json")
    return [(EXEC, c["expect_stored"].encode("utf-8"), c) for c in g["execution_vcs"]] + \
           [(WF, c["expect_stored"].encode("utf-8"), c) for c in g["workflow_vcs"]]


def test_spellings_keep_number_tokens():
    for _, doc, _ in _golden_docs():
        for how in SPELLINGS:
            s = spell(doc, how)
            assert sorted(re.findall(rb"(?<=[:\[,\s])-?\d[\d.eE+-]*", _strip_strings(s))) == \
                sorted(re.findall(rb"(?<=[:\[,\s])-?\d[\d.eE+-]*", _strip_strings(doc))), how


def _strip_strings(b):
    return re.sub(rb'"(?:[^"\\]|\\.)*"', b'""', b)


@pytest.mark.parametrize("how", sorted(SPELLINGS))
def test_golden_spellings(vcj, how):
    """Each golden document in each client spelling: the invariant holds; the 14 whose metadata holds no fraction or exponent are
    never declined, and those without \\ufffd come out VALID with the reference's signing bytes and signature."""
    accepted = 0
    for kind, doc, c in _golden_docs():
        s = spell(doc, how)
        assert s != doc or how == "compact"                  # a document with nothing to escape is already compact ASCII
        st, msg = check(vcj, kind, s)
        if _FLOATISH.search(_metadata(doc)):
            continue
        assert st != HOST, (c["id"], s[:200])
        accepted += 1
        if b"\\ufffd" not in doc:
            assert st == VALID
            assert msg == c["expect_canonical"].encode("utf-8")
            assert run(vcj, kind, s)[2].hex() == c["expect_sig"]
    assert accepted == 14


def _respell_random(rng, v, protect=False):
    """Whitespace runs at every token boundary; each string character possibly written as an escape (\\uXXXX in either case, a
    surrogate pair, \\/).  Member names, metadata keys, issuer and proofValue keep their bytes."""
    def ws():
        return "".join(rng.choice([" ", "\t", "\n", "\r"]) for _ in range(rng.integers(0, 3) if rng.random() < 0.7 else 0))

    def s_esc(s):
        out = []
        for ch in s:
            r = rng.random()
            cp = ord(ch)
            if r < 0.15 and cp >= 0x10000:
                hi, lo = 0xD800 + ((cp - 0x10000) >> 10), 0xDC00 + ((cp - 0x10000) & 0x3FF)
                out.append(("\\u%04x\\u%04x" if rng.random() < 0.5 else "\\u%04X\\u%04X") % (hi, lo))
            elif r < 0.15:
                out.append(("\\u%04x" if rng.random() < 0.5 else "\\u%04X") % cp)
            elif ch == "/" and r < 0.5:
                out.append("\\/")
            else:
                out.append(json.dumps(ch, ensure_ascii=False)[1:-1])
        return '"' + "".join(out) + '"'

    def plain(s):
        return json.dumps(s, ensure_ascii=False)

    def w(x, keep):
        if isinstance(x, Num):
            return str(x)
        if isinstance(x, str):
            return plain(x) if keep else s_esc(x)
        if x is None or isinstance(x, bool):
            return json.dumps(x)
        if isinstance(x, tuple):
            parts = [ws() + plain(k) + ws() + ":" + ws() + w(y, k in ("issuer", "proofValue")) + ws() for k, y in x[1]]
            return "{" + (",".join(parts) if parts else ws()) + "}"
        parts = [ws() + w(y, False) + ws() for y in x]
        return "[" + (",".join(parts) if parts else ws()) + "]"
    return (ws() + w(v, False) + ws()).encode("utf-8")


def test_random_documents_respelled(vcj):
    """The random issued documents of the stored-document tests, each re-spelled at random: the invariant holds, and over 400 of the
    600 are accepted."""
    rng = np.random.default_rng(0xAFD0)
    wrng = np.random.default_rng(0xAFE0)
    accepted = 0
    for i in range(600):
        sig = rng.integers(0, 256, 64, dtype=np.uint8).tobytes()
        kind = EXEC if i % 2 == 0 else WF
        _, doc = (_rand_exec if kind == EXEC else _rand_wf)(rng, sig)
        s = _respell_random(wrng, parse_keep(doc))
        st, _ = check(vcj, kind, s)
        accepted += st != HOST
    assert accepted > 400, accepted


def _with_meta(doc, text):
    return doc.replace(b'"metadata":{', b'"metadata":{' + text, 1)


def test_number_tokens(vcj):
    """Re-spellings keep every number token (above).  The other way on purpose: -0 in metadata through plain json.loads / json.dumps
    becomes 0, as JSON.stringify writes it; the message is then the mirror's, with 0."""
    kind, doc, _ = _golden_docs()[0]
    neg = _with_meta(doc, b'"!":-0,')
    st, msg = check(vcj, kind, neg)
    assert st == VALID and b'"!":-0,' in msg
    plain = json.dumps(json.loads(neg)).encode()
    assert b'"!": 0,' in plain
    st, msg = check(vcj, kind, plain)
    assert st == VALID and b'"!":0,' in msg and b'"!":-0' not in msg


def _indent2_sources():
    docs = _golden_docs()
    return [(docs[0][0], spell(docs[0][1], "indent2")), (docs[10][0], spell(docs[10][1], "js_pretty"))]


@pytest.mark.parametrize("which", range(2))
def test_every_single_byte_mutation(vcj, which):
    """Every single-byte deletion, duplication and substitution of two pretty-printed documents: each verdict is exact."""
    kind, doc = _indent2_sources()[which]
    assert run(vcj, kind, doc)[0] == VALID
    accepted = 0
    for i in range(len(doc)):
        for m in (doc[:i] + doc[i + 1:], doc[:i + 1] + doc[i:]):
            accepted += check(vcj, kind, m)[0] != HOST
        for b in SUBS + [b"\t", b"\n", b"\r"]:
            if doc[i:i + 1] != b:
                accepted += check(vcj, kind, doc[:i] + b + doc[i + 1:])[0] != HOST
    assert accepted > len(doc)


def _declines(doc, kind):
    s = doc.decode("utf-8")
    yield "reordered", _swap_members(s, '"id"', '"issuer"')
    yield "unknown", s.replace('"issuanceDate"', '"extra": 1,\n  "issuanceDate"', 1)
    yield "duplicate", s.replace('"issuanceDate": "', '"issuanceDate": "x",\n  "issuanceDate": "', 1)
    yield "case variant", s.replace('"issuanceDate"', '"IssuanceDate"', 1)
    yield "escaped name", s.replace('"issuanceDate"', '"issuance\\u0044ate"', 1)
    yield "bom", "\ufeff" + s
    yield "nan", _meta_s(s, '"!": NaN, ')
    yield "trailing comma", re.sub(r'"(\s*)\]', r'",\1]', s, count=1)
    yield "null string", re.sub(r'"sessionId": "[^"]*"', '"sessionId": null', s, count=1)
    yield "null in list", s.replace('"VerifiableCredential"', 'null', 1)
    yield "unsorted keys", _meta_s(s, '"b": 1, "a": 2, ')
    yield "js integer keys first", _meta_s(s, '"9": 2, "10": 1, ')
    yield "duplicate keys", _meta_s(s, '"a": 1, "a": 1, ')
    yield "escaped key", _meta_s(s, '"\\u0021": 1, ')
    yield "too deep", _meta_s(s, '"!": ' + "[" * 9 + "]" * 9 + ", ")
    yield "fraction in metadata", _meta_s(s, '"!": 1.0, ')
    yield "exponent in metadata", _meta_s(s, '"!": 1e2, ')
    yield "long metadata integer", _meta_s(s, '"!": 1234567890123456, ')
    yield "leading zero", _meta_s(s, '"!": 01, ')
    yield "raw control byte", s.replace('"issuanceDate": "', '"issuanceDate": "\x01', 1)
    yield "lone high surrogate", s.replace('"issuanceDate": "', '"issuanceDate": "\\ud83d', 1)
    yield "lone low surrogate", s.replace('"issuanceDate": "', '"issuanceDate": "\\ude00', 1)
    yield "escape in issuer", s.replace('"issuer": "did', '"issuer": "\\u0064id', 1)
    yield "escape in proofValue", s.replace('"proofValue": "', '"proofValue": "\\/', 1)
    if kind == EXEC:
        yield "1.0 in an int member", re.sub(r'"durationMs": \d+', '"durationMs": 1.0', s, count=1)
        yield "1e2 in an int member", re.sub(r'"durationMs": \d+', '"durationMs": 1e2', s, count=1)
        yield "int64 overflow", re.sub(r'"durationMs": \d+', '"durationMs": 9223372036854775808', s, count=1)
        yield "missing member", re.sub(r',\s*"sessionId": "[^"]*"', "", s, count=1)
        yield "errorMessage null", re.sub(r'("status": "[^"]*")', r'\1, "errorMessage": null', s, count=1)


def _swap_members(s, a, b):
    i, j = s.index(a + ":"), s.index(b + ":")
    k = s.index(",", j)
    first, second = s[i:s.index(",", i)], s[j:k]
    return s[:i] + second + s[s.index(",", i):j] + first + s[k:]


def _meta_s(s, text):
    return re.sub(r'"metadata": \{', lambda m: m.group(0) + text, s, count=1)


def test_targeted_declines(vcj):
    for kind, doc, _ in (_golden_docs()[0], _golden_docs()[10]):
        s = spell(doc, "indent2")
        assert run(vcj, kind, s)[0] == VALID
        for what, t in _declines(s, kind):
            raw = t.encode("utf-8", "surrogatepass")
            assert raw != s, what
            assert run(vcj, kind, raw)[0] == HOST, (what, raw[:300])
    # raw truncated UTF-8 (Go writes one U+FFFD per byte; the mirror folds the sequence into one: left to the host)
    kind, doc, _ = _golden_docs()[0]
    assert run(vcj, kind, doc.replace(b'"issuanceDate":"', b'"issuanceDate":"\xe6\x97', 1))[0] == HOST
    assert run(vcj, kind, doc.replace(b'"issuanceDate":"', b'"issuanceDate":"\xff', 1))[0] == HOST


def _pad_to(vcj, kind, doc, extra):
    """doc with `extra` raw '<' added to the proof's type (dropped from the message) and raw '<' in the id (6 bytes in the message
    each): returns the document whose message is exactly len(doc) + extra bytes long, extra <= 0 accepted."""
    st, msg, _, _ = run(vcj, kind, doc)
    slack = len(doc) - len(msg)
    k = slack // 5 + 1                                   # k raw '<' in the id grow the message by 5 k more than the document
    d = doc.replace(b'"id":"', b'"id":"' + b"<" * k, 1)
    over = len(msg) + 6 * k - len(d)                     # > 0: the message is this much longer than the document
    d = d.replace(b'"proof":{"type":"', b'"proof":{"type":"' + b"x" * (over - extra), 1)
    return d


def test_targeted_accepts(vcj):
    kind, doc, c = _golden_docs()[0]
    s = spell(doc, "indent2")
    cases = {
        "-0 in durationMs": re.sub(rb'"durationMs": \d+', b'"durationMs": -0', s, count=1),
        "raw < and U+2028": s.replace(b'"issuanceDate": "', b'"issuanceDate": "<\xe2\x80\xa8', 1),
        "uppercase escape": s.replace(b'"issuanceDate": "', b'"issuanceDate": "\\u003C', 1),
        "DEL escape": s.replace(b'"issuanceDate": "', b'"issuanceDate": "\\u007f', 1),
        "empty errorMessage": re.sub(rb'("status": "[^"]*")', rb'\1, "errorMessage": ""', s, count=1),
        "U+FFFD escape": s.replace(b'"issuanceDate": "', b'"issuanceDate": "\\ufffd', 1),
    }
    for what, t in cases.items():
        st, msg = check(vcj, kind, t)
        assert st in (VALID,), what
    assert b'"durationMs":0,' in check(vcj, kind, cases["-0 in durationMs"])[1]
    assert b'"issuanceDate":"\\u003c\\u2028' in check(vcj, kind, cases["raw < and U+2028"])[1]
    assert b'"issuanceDate":"\\u003c' in check(vcj, kind, cases["uppercase escape"])[1]
    assert b'"issuanceDate":"\x7f' in check(vcj, kind, cases["DEL escape"])[1]
    assert check(vcj, kind, cases["empty errorMessage"])[1] == c["expect_canonical"].encode()
    assert b'"issuanceDate":"\xef\xbf\xbd' in check(vcj, kind, cases["U+FFFD escape"])[1]
    wkind, wdoc, _ = _golden_docs()[10]
    ws = spell(wdoc, "indent2")
    assert b'"endTime"' not in ws
    null_end = re.sub(rb'("startTime": "[^"]*")', rb'\1, "endTime": null', ws, count=1)
    empty_end = re.sub(rb'("startTime": "[^"]*")', rb'\1, "endTime": ""', ws, count=1)
    assert check(vcj, wkind, null_end)[1] == check(vcj, wkind, ws)[1]
    assert b',"endTime":"",' in check(vcj, wkind, empty_end)[1]
    # the length bound: a message exactly as long as its document is accepted, one byte longer is not
    at = _pad_to(vcj, kind, doc, 0)
    st, msg = check(vcj, kind, at)
    assert st != HOST and len(msg) == len(at)
    past = _pad_to(vcj, kind, doc, 1)
    assert run(vcj, kind, past)[0] == HOST
    assert go_unmarshal_vc(past, kind) and len(mirror_message(go_unmarshal_vc(past, kind), kind)) == len(past) + 1


def test_length_bound_is_decided_on_the_full_count(vcj):
    """A document of 0.75 GB whose id is 750 M raw '<': the canonical prefix is 4.5 GB (each '<' becomes six bytes), past 2^32.  The
    bound is decided on the 64-bit count, so the walk declines it; a 32-bit count would wrap to about 0.2 GB and pass."""
    kind, doc, _ = _golden_docs()[0]
    k = doc.index(b'"id":"') + len(b'"id":"')
    n_lt = 750_000_000
    total = len(doc) + n_lt
    buf = (C.c_uint8 * total)()
    C.memmove(buf, doc, k)
    C.memset(C.addressof(buf) + k, ord("<"), n_lt)
    C.memmove(C.addressof(buf) + k + n_lt, doc[k:], len(doc) - k)
    count = C.c_uint64()
    assert vcj.hs_vcj_sizes(kind, buf, C.c_uint64(total), C.byref(count)) == 0
    assert count.value > 1 << 32 and (count.value & 0xffffffff) + TAIL <= total        # the wrapped count would have passed
    del buf


def test_code_point_escaper_matches_go_json_escape(vcj):
    """vcj_put_cp (code points) against go_json_escape (bytes) for every class: U+0000-U+00FF, U+07FF / U+0800, U+2027-U+202A,
    U+FFFD, U+10FFFF and a few more."""
    a, b = (C.c_uint8 * 8)(), (C.c_uint8 * 64)()
    cps = list(range(0x100)) + [0x7FF, 0x800, 0x2027, 0x2028, 0x2029, 0x202A, 0xD7FF, 0xE000, 0xFFFD, 0xFFFF, 0x10000, 0x1F600, 0x10FFFF]
    for cp in cps:
        u = chr(cp).encode("utf-8")
        n = vcj.hs_vcj_put_cp(cp, a)
        m = vcj.hs_go_json_escape(u, C.c_uint64(len(u)), b)
        assert bytes(a)[:n] == bytes(b)[:m] == GJ.string(chr(cp))[1:-1].encode("utf-8"), hex(cp)
