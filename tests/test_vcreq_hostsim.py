"""The request bind and response writer (agentfield_b200/csrc/afc_vcreq.cuh), compiled for the CPU (tests/hostsim/hostsim_vcreq.cpp) together
with the json-verify walk it hands the vc_document to, against the oracle (tests/verify_request_oracle.py).  For every body the CPU build
gives HOST or exactly the oracle's (state, body).  Inputs: every truncation of SDK-shaped (json.dumps), compact UI-shaped (JSON.stringify)
and 2-space-pretty request bodies around the golden execution credentials, every single-byte deletion and substitution of those bodies,
and envelopes with extra members, duplicate and re-cased keys, trailing bytes, leading whitespace, a BOM, null and non-object values.
Coverage: the realistic shapes never go to the host, and syntax errors reach BAD_REQUEST."""
import ctypes as C
import json
import os
import subprocess

import pytest

import verify_request_oracle as O
from agentfield_b200 import respell as R
from conftest import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VRB_BAD, VRB_NO_DOC, VRB_NULL_DOC, VRB_HOST, VRB_OBJECT = 0, 1, 2, 3, 4
VC_INVALID, VC_VALID, VC_HOST, VC_UNRESOLVED, VC_BAD_ENCODING = 0, 1, 2, 3, 4


def build_cpu_request(tmp_path_factory):
    """TEST-ONLY CPU build of afc_vcreq.cuh (tests/hostsim/hostsim_vcreq.cpp), compiled into a temporary directory."""
    out = str(tmp_path_factory.mktemp("vrqsim") / "libafc_vrqsim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_vcreq.cpp")])
    lib = C.CDLL(out)
    lib.hs_vrq_bind.restype = C.c_uint32
    lib.hs_vrq_fixed.restype = C.c_uint64
    return lib


@pytest.fixture(scope="module")
def vrq(tmp_path_factory):
    return build_cpu_request(tmp_path_factory)


def cpu_answer(lib, body, registry):
    """What the device pipeline computes for one body: (state, response bytes); the issuer lookup and the signature check, which the
    device does with the key set's table and the keyed verify, are done here with the registry and the oracle's ed25519.Verify."""
    span = (C.c_uint32 * 2)()
    kind = lib.hs_vrq_bind(body, C.c_uint64(len(body)), span)
    doc, status = b"", VC_HOST
    fields, at = (C.c_uint32 * 4)(), C.c_uint32()
    if kind == VRB_OBJECT:
        doc = body[span[0]:span[0] + span[1]]
        msg, ml, sig = (C.c_uint8 * (len(doc) + 64))(), C.c_uint64(), (C.c_uint8 * 64)()
        status = lib.hs_vrq_doc(doc, C.c_uint64(len(doc)), msg, C.byref(ml), sig, fields, C.byref(at))
        if status != VC_HOST:
            iss = doc[fields[0]:fields[0] + fields[1]].decode("utf-8")
            if iss not in registry:
                status = VC_UNRESOLVED
            elif status == VC_VALID:
                status = VC_VALID if O._verify(registry[iss], bytes(msg)[:ml.value], bytes(sig)) else VC_INVALID
    elif kind == VRB_NULL_DOC and "" in registry:
        kind = VRB_HOST
    out, olen = (C.c_uint8 * (lib.hs_vrq_fixed() + 6 * len(body) + 64))(), C.c_uint64()
    st = lib.hs_vrq_body(kind, status, doc, fields, at, out, C.byref(olen))
    assert st >= 0, body[:200]
    return st, bytes(out)[:olen.value]


def check(lib, body, registry):
    """Asserts the module's invariant for one body; returns the state (O.HOST for a declined one)."""
    got = cpu_answer(lib, body, registry)
    if got[0] == O.HOST:
        assert got[1] == b""
        return O.HOST
    want = O.answer(body, registry)
    assert want is not None, ("answered a body the oracle leaves open", body[:300])
    assert got == want, (got, want, body[:300])
    return got[0]


def registry():
    g = golden("go_cases.json")
    return {c["issuer"]: bytes.fromhex(c["pk"]) for c in g["execution_vcs"]}


def golden_docs():
    return [c["expect_stored"].encode("utf-8") for c in golden("go_cases.json")["execution_vcs"]]


def realistic_docs():
    """The golden documents whose metadata holds strings and integers only: floats in metadata are left to the host by the json-verify
    path, so requests around the others are HOST by design."""
    return [d for d in golden_docs() if not any(t in d for t in (b"1.5", b"2.5", b"1e", b"67000"))]


def _wrap(doc):
    """{"vc_document": doc} with every number token of doc kept as it stood (agentfield_b200.respell)."""
    return ("obj", [("vc_document", R.parse_keep(doc))])


def sdk_body(doc):
    """requests.post(json={"vc_document": vc}) of the Python SDK: json.dumps with its default separators, ASCII escapes."""
    return R.SPELLINGS["dumps"](_wrap(doc)).encode("utf-8")


def ui_body(doc):
    """JSON.stringify({vc_document}) of the web UI: compact, non-ASCII as it is."""
    return R.write(_wrap(doc), esc=R._esc_js).encode("utf-8")


def pretty_body(doc):
    return R.SPELLINGS["indent2"](_wrap(doc)).encode("utf-8")


SHAPES = (sdk_body, ui_body, pretty_body)


def test_realistic_shapes_are_answered(vrq):
    reg = registry()
    docs = realistic_docs()
    assert len(docs) >= 4
    for doc in docs:
        for shape in SHAPES:
            body = shape(doc)
            assert check(vrq, body, reg) == O.OK, body[:200]
            assert b'"valid":true' in cpu_answer(vrq, body, reg)[1]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda f: f.__name__)
def test_every_truncation(vrq, shape):
    reg = registry()
    body = shape(realistic_docs()[0])
    states = [check(vrq, body[:i], reg) for i in range(len(body))]
    assert O.HOST not in states
    assert states.count(O.BAD_REQUEST) == len(body)          # a cut body is never a whole object


SUBS = [b'"', b"\\", b"A", b"}", b"\x01", b" "]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda f: f.__name__)
def test_every_single_byte_mutation(vrq, shape):
    reg = registry()
    body = shape(realistic_docs()[1])
    counts = {O.OK: 0, O.BAD_REQUEST: 0, O.HOST: 0}
    for i in range(len(body)):
        for m in [body[:i] + body[i + 1:]] + [body[:i] + s + body[i + 1:] for s in SUBS if body[i:i + 1] != s]:
            st = check(vrq, m, reg)
            counts[st] += 1
            if st == O.HOST:
                # a declined body is one the walk declines: never a plain syntax error
                assert O.bind(m)[0] != "bad", m[:300]
    assert counts[O.BAD_REQUEST] > counts[O.HOST] and counts[O.OK] > 0, counts


def test_envelopes(vrq):
    reg = registry()
    doc = realistic_docs()[2]
    compact = R.write(R.parse_keep(doc)).encode("utf-8")
    other = realistic_docs()[3]
    cases = {
        b'{"vc_document":' + doc + b'}': O.OK,
        b'{"a":1,"b":[true,null,{"c":"\\u0041"}],"vc_document":' + doc + b',"z":-1.5e3}': O.OK,
        b'{"VC_Document":' + doc + b'}': O.OK,
        b'{"vc_document":' + other + b',"Vc_Document":' + doc + b'}': O.OK,            # the last match wins
        b'{"vc_document":' + doc + b',"vc_document":null}': O.OK,
        b'{"vc_document":' + doc + b'} trailing [garbage': O.OK,
        b'{"vc_document":' + doc + b'}{"vc_document":1}': O.OK,
        b' \t\r\n{"vc_document":' + compact + b'}': O.OK,
        b'\xef\xbb\xbf{"vc_document":' + doc + b'}': O.BAD_REQUEST,
        b'{"vc_document":' + doc + b',"x":01}': O.BAD_REQUEST,                        # a syntax error after the member still fails
        b'{"vc_document":' + doc + b',"x":"\x01"}': O.BAD_REQUEST,
        b'{"vc_document":' + doc + b',"x":"\\q"}': O.BAD_REQUEST,
        b'{"vc_document":' + doc + b',}': O.BAD_REQUEST,
        b'': O.BAD_REQUEST, b'   ': O.BAD_REQUEST, b'[]': O.BAD_REQUEST, b'"x"': O.BAD_REQUEST, b'12': O.BAD_REQUEST,
        b'true': O.BAD_REQUEST, b'false': O.BAD_REQUEST, b'nul': O.BAD_REQUEST, b'{': O.BAD_REQUEST,
        b'null': O.OK, b'null x': O.OK, b'{}': O.OK, b'{"vc_documents":{}}': O.OK, b'{"vc_document":null}': O.OK,
        b'{"vc_document":{}}': O.HOST,                                                   # the walk declines missing members
        b'{"vc_document":"x"}': O.HOST, b'{"vc_document":[1]}': O.HOST, b'{"vc_document":1}': O.HOST, b'{"vc_document":true}': O.HOST,
        b'{"vc_\\u0064ocument":' + doc + b'}': O.HOST, b'{"\xc3\xa9":1}': O.HOST,
        b'{"a":' + b"[" * 70 + b"]" * 70 + b'}': O.HOST,
        b'{"a":' + b"[" * 70 + b"]" * 69 + b'}': O.HOST,
    }
    for body, want in cases.items():
        got = check(vrq, body, reg)
        assert got == want, (want, got, body[:200])
    assert cpu_answer(vrq, b'{"vc_document":null}', reg)[1] == \
        b'{"valid":false,"error":"failed to resolve issuer DID: DID not found: "}'
    assert cpu_answer(vrq, b'{}', reg)[1] == b'{"valid":false,"error":"failed to parse VC document: unexpected end of JSON input"}'
    # the empty DID in the registry: the host runs the zero document's verify
    assert cpu_answer(vrq, b'{"vc_document":null}', dict(reg, **{"": bytes(32)}))[0] == O.HOST


def test_verdict_rows(vrq):
    """Each verdict of an object vc_document: unknown issuer, a bad base64 character or length, a wrong signature, an escaped issuance date."""
    reg = registry()
    doc = json.loads(realistic_docs()[0])
    pv = doc["proof"]["proofValue"]
    rows = []
    for iss, p, date in ((doc["issuer"], pv, doc["issuanceDate"]), ("did:key:z6MkUnknown<&>", pv, doc["issuanceDate"]),
                         (doc["issuer"], pv[:10] + "+" + pv[11:], doc["issuanceDate"]), (doc["issuer"], pv + "AAA", doc["issuanceDate"]),
                         (doc["issuer"], pv[:-2] + ("B" if pv[-2] != "B" else "C") + pv[-1], doc["issuanceDate"]),
                         (doc["issuer"], pv[:-4], doc["issuanceDate"]), (doc["issuer"], pv, doc["issuanceDate"] + " <x>")):
        d = dict(doc, issuer=iss, issuanceDate=date, proof=dict(doc["proof"], proofValue=p))
        body = json.dumps({"vc_document": d}).encode()
        assert check(vrq, body, reg) == O.OK, body[:200]
        rows.append(cpu_answer(vrq, body, reg)[1])
    assert b'"valid":true' in rows[0]
    assert rows[1] == b'{"valid":false,"error":"failed to resolve issuer DID: DID not found: did:key:z6MkUnknown\\u003c\\u0026\\u003e"}'
    assert rows[2].endswith(b'illegal base64 data at input byte 10"}')
    assert rows[3].endswith(b'illegal base64 data at input byte 88"}')
    assert rows[4] == rows[5] == b'{"valid":false,"message":"Invalid signature"}'
    assert rows[6] == b'{"valid":false,"message":"Invalid signature"}'


def test_b64_error_index_skips_newlines():
    assert O.b64_error_at(b"AAAA") is None
    assert O.b64_error_at(b"AAAAA") == 4
    assert O.b64_error_at(b"AAAAA\n") == 5
    assert O.b64_error_at(b"AA\r\nAA") is None
    assert O.b64_error_at(b"AA\nA*") == 4


def test_golden_request_cases(vrq):
    """tests/golden/verify_request_cases.json (written by make_verify_request_cases.py, pinned against Go by baseline/go/gen_golden_test.go):
    the oracle gives every expectation, and the CPU build gives it or HOST."""
    g = golden("verify_request_cases.json")
    reg = {r["did"]: bytes.fromhex(r["pk"]) for r in g["registry"]}
    host = 0
    for c in g["cases"]:
        body = bytes.fromhex(c["body_hex"])
        want = (O.OK if c["expect_status"] == 200 else O.BAD_REQUEST, c["expect_body"].encode("utf-8"))
        assert O.answer(body, reg) == want, c["name"]
        got = cpu_answer(vrq, body, reg)
        host += got[0] == O.HOST
        assert got[0] == O.HOST or got == want, (c["name"], got, want)
    assert host <= 6
