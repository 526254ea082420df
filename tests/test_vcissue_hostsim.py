"""The issuing routines (agentfield_b200/csrc/afc_vcissue.cuh), compiled for the CPU (tests/hostsim/hostsim_vcissue.cpp), against the
oracle: hashData (oracle/go_hash.py) for every payload length and alignment, and the signing message and stored document of
GenerateExecutionVC (oracle/ref_vc.py) for strings of every escape class, error messages cut inside runes, extreme durations, hashing
off and the golden Go cases.  Also checks that afc_vc_issue_bound (libafcrypto.so, host arithmetic only) is at least the real size."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import golden
from oracle import go_hash as H, ref_vc as RV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COLUMNS = ("vc_id", "caller_did", "issuance_date", "execution_id", "workflow_id", "session_id", "caller_type", "agent_node_did", "target_did",
           "function_name", "timestamp", "status", "error_message", "proof_created")
PLACEHOLDER = "A" * 86


@pytest.fixture(scope="module")
def vci(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("vcisim") / "libafc_vcisim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_vcissue.cpp")])
    return C.CDLL(out)


def hashdata(vci, data, align=0):
    """hashData of one payload (None = nil) placed at `align` bytes past a 16-byte boundary, bytes after it non-zero."""
    raw = b"" if data is None else bytes(data)
    buf = np.full(len(raw) + align + 64, 0xA5, dtype=np.uint8)
    base = (-buf.ctypes.data) % 16
    buf[base + align:base + align + len(raw)] = np.frombuffer(raw, dtype=np.uint8)
    out = (C.c_uint8 * 43)()
    vci.hs_vci_hashdata(C.c_void_p(buf.ctypes.data + base + align), C.c_uint64(len(raw)), int(data is None), out)
    return bytes(out).decode()


def expect_hash(data):
    return H.hash_data(H.marshal_data_or_null(data))


def pack_columns(values):
    raw = [v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v) for v in values]
    off = np.zeros(len(raw) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(v) for v in raw])
    return np.frombuffer(b"".join(raw) + b"\0" * 8, dtype=np.uint8).copy(), off


def device_doc(vci, req, hashes):
    """(signing message, stored document with the proofValue placeholder) as the fill pass writes them."""
    cols, off = pack_columns([req[k] for k in COLUMNS])
    ml, dl = C.c_uint64(), C.c_uint64()
    h = None if hashes is None else np.frombuffer((hashes[0] + hashes[1]).encode(), dtype=np.uint8).copy()
    assert vci.hs_vci_sizes(cols.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), C.c_int64(req["duration_ms"]),
                            None if h is None else h.ctypes.data_as(C.c_void_p), C.byref(ml), C.byref(dl)) == 0
    msg, doc = (C.c_uint8 * (ml.value + 32))(), (C.c_uint8 * (dl.value + 32))()
    assert vci.hs_vci_doc(cols.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), C.c_int64(req["duration_ms"]),
                          None if h is None else h.ctypes.data_as(C.c_void_p), msg, C.byref(ml), doc, C.byref(dl)) == 0
    return bytes(msg)[:ml.value], bytes(doc)[:dl.value]


def go_str(v):
    """A column as the oracle's Go string (invalid UTF-8 bytes as its marker)."""
    return RV._go_bytes_as_str(v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v))


def oracle_doc(req, hashes):
    """(signing message, stored document with the placeholder proofValue) from oracle/ref_vc.py."""
    raw_em = req["error_message"].encode("utf-8", "surrogatepass") if isinstance(req["error_message"], str) else bytes(req["error_message"])
    em = RV._go_bytes_as_str(raw_em[:500]) + "...[truncated]" if len(raw_em) > 500 else RV._go_bytes_as_str(raw_em)
    r = {k: go_str(req[k]) for k in COLUMNS if k != "error_message"}
    r["duration_ms"] = int(req["duration_ms"])
    r["error_message"] = None
    ih, oh = hashes if hashes is not None else ("", "")

    def doc(proof):
        d = RV.vc_document(r, ih, oh, proof)
        if em:
            d["credentialSubject"]["execution"]["errorMessage"] = em
        return RV.go_marshal(d)
    proof = {"type": "Ed25519Signature2020", "created": r["proof_created"], "verificationMethod": "%s#key-1" % r["caller_did"],
             "proofPurpose": "assertionMethod", "proofValue": PLACEHOLDER}
    return doc(None), doc(proof)


def base_request(**kw):
    r = {"vc_id": "5f0c5b4e-6a3c-4f7e-9b1a-2d3c4e5f6a7b", "caller_did": "did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A",
         "issuance_date": "2026-09-21T06:00:00Z", "execution_id": "exec_0001", "workflow_id": "wf_0001", "session_id": "sess_0001",
         "caller_type": "agent", "agent_node_did": "did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A", "target_did": "did:key:zTarget",
         "function_name": "summarize", "timestamp": "2026-09-21T06:00:00.123456789Z", "status": "succeeded", "error_message": "",
         "proof_created": "2026-09-21T06:00:01Z", "duration_ms": 1234}
    r.update(kw)
    return r


def check(vci, req, hashes=("LcOQZrtCEWLLHIf8LxBLHqxeuQhh29gbI2UNPfFHENM", "dCNOmK_nSY-12vHzasLXiswzlGT5UHA7jAGYkvmCuQs")):
    got = device_doc(vci, req, hashes)
    want = oracle_doc(req, hashes)
    assert got[0] == want[0], (got[0], want[0])
    assert got[1] == want[1], (got[1], want[1])


# ---- hashData
def test_hashdata_every_length_and_alignment(vci):
    rng = np.random.default_rng(1)
    for n in range(0, 301):
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        for a in range(16):
            assert hashdata(vci, data, a) == expect_hash(data), (n, a)


def test_hashdata_block_boundaries_nil_and_empty(vci):
    rng = np.random.default_rng(2)
    assert hashdata(vci, None) == expect_hash(None) == H.b64url_nopad(H.sha256(b"null"))
    assert hashdata(vci, b"") == expect_hash(b"") == H.b64url_nopad(H.sha256(b'""'))
    for k in range(1, 90):
        for d in (-2, -1, 0, 1, 2):
            n = 48 * k + d
            data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
            for a in (0, 3, 8):
                assert hashdata(vci, data, a) == expect_hash(data), (n, a)


# ---- documents
ESCAPE_CLASSES = ["plain", "quote\"back\\slash", "ctl\x00\x01\x08\x0c\n\r\t\x1f\x7f", "html<>&", "ls ps ", "utf8 é ✓ 𝄞",
                  b"bad\x80\xbf", b"\xc0\xaf overlong", b"\xed\xa0\x80 surrogate", b"\xf4\x90\x80\x80 too big", b"cut \xe2\x82", b"\xff\xfe",
                  "", "a" * 300]


def test_documents_every_escape_class(vci):
    for k in COLUMNS:
        for v in ESCAPE_CLASSES:
            check(vci, base_request(**{k: v}))


def test_documents_random_strings(vci):
    rng = np.random.default_rng(3)
    pieces = [b"a", b"Z", b"0", b"\"", b"\\", b"<", b">", b"&", b"\x00", b"\x1f", b"\n", b"\x7f", " ".encode(), "é".encode(), "✓".encode(),
              "𝄞".encode(), b"\x80", b"\xff", b"\xe2\x82", b"\xed\xa0\x80"]
    for _ in range(300):
        req = base_request()
        for k in COLUMNS:
            if rng.random() < 0.5:
                req[k] = b"".join(pieces[j] for j in rng.integers(0, len(pieces), int(rng.integers(0, 40))))
        req["duration_ms"] = int(rng.integers(-2**63, 2**63 - 1, dtype=np.int64))
        check(vci, req)


def test_error_message_cut_inside_runes(vci):
    for rune in ("é", "✓", "𝄞"):
        rb = rune.encode()
        for total in (499, 500, 501, 502, 503, 504, 520):
            for shift in range(len(rb)):
                pre = "x" * (500 - shift - 1)                       # the rune starts at byte 499 - shift: every cut position inside it
                msg = (pre + rune * 8)[:total] if len((pre + rune * 8).encode()) >= total else pre + rune * 8
                raw = msg.encode()[:total]
                check(vci, base_request(error_message=raw))
                check(vci, base_request(error_message=raw + b"<&>\n"))
    for n in (499, 500, 501):
        check(vci, base_request(error_message="e" * n))


def test_durations(vci):
    for d in (0, 1, -1, 9, 10, -10, 999999, 10**18, -10**18, 10**18 - 1, 2**63 - 1, -2**63, -2**63 + 1, 1234567890123456789):
        check(vci, base_request(duration_ms=d))


def test_hash_data_off(vci):
    check(vci, base_request(), hashes=None)
    check(vci, base_request(error_message="boom"), hashes=None)


def test_proof_value(vci):
    rng = np.random.default_rng(4)
    for _ in range(200):
        sig = rng.integers(0, 256, 64, dtype=np.uint8).tobytes()
        a, b = (C.c_uint8 * 86)(), (C.c_uint8 * 86)()
        vci.hs_vci_proof(sig, a, b)
        assert bytes(a) == bytes(b) == H.b64url_nopad(sig).encode()


def _with_issued_metadata(text):
    """A golden document with its metadata replaced by the one createVCDocument writes (the golden cases vary it; issuing does not)."""
    raw = text.encode("utf-8", "surrogatepass")
    a = raw.rindex(b'"metadata":') + len(b'"metadata":')
    b = raw.index(b'}},"proof":', a)
    return raw[:a] + b'{"agentfield_version":"1.0.0","vc_version":"1.0"}' + raw[b:]


def test_golden_execution_vcs(vci):
    """The reference's own output for every golden execution VC with the @context and type createVCDocument writes: the signing bytes,
    and the stored document with the golden signature as proofValue (metadata set to the issued one)."""
    used = 0
    for c in golden("go_cases.json")["execution_vcs"]:
        if (c["context"] != ["https://www.w3.org/2018/credentials/v1", "https://agentfield.example.com/contexts/execution/v1"]
                or c["type"] != ["VerifiableCredential", "AgentFieldExecutionCredential"]):
            continue
        assert c["id"].startswith("urn:agentfield:vc:") and c["issuer"] == c["caller"]["did"] and c["target"]["agent_node_did"] == c["caller"]["agent_node_did"]
        assert (c["input_hash"], c["output_hash"]) == (c["input_data_hash"], c["output_data_hash"])
        req = {"vc_id": c["id"][len("urn:agentfield:vc:"):], "caller_did": c["issuer"], "issuance_date": c["issuance_date"],
               "execution_id": c["execution_id"], "workflow_id": c["workflow_id"], "session_id": c["session_id"], "caller_type": c["caller"]["type"],
               "agent_node_did": c["caller"]["agent_node_did"], "target_did": c["target"]["did"], "function_name": c["target"]["function_name"],
               "timestamp": c["timestamp"], "status": c["status"], "error_message": c["error_message_input"], "proof_created": c["proof_created"],
               "duration_ms": c["duration_ms"]}
        msg, doc = device_doc(vci, req, (c["input_hash"], c["output_hash"]))
        assert msg == _with_issued_metadata(c["expect_canonical"])
        a, b = (C.c_uint8 * 86)(), (C.c_uint8 * 86)()
        vci.hs_vci_proof(bytes.fromhex(c["expect_sig"]), a, b)
        stored = doc[:len(doc) - 89] + bytes(a) + doc[len(doc) - 3:]
        assert stored == _with_issued_metadata(c["expect_stored"])
        used += 1
    assert used == 8


# ---- the bound
def test_bound_covers_worst_case_and_random_strings(vci):
    from agentfield_b200 import _abi
    lib = _abi.load()
    lib.afc_vc_issue_bound.restype = C.c_uint64
    rng = np.random.default_rng(5)
    worst = [bytes(range(32)) * 20, b"\xff" * 700, b"<" * 600, " ".encode() * 200, b"\x80" * 999]
    cases = [{k: w for k in COLUMNS} for w in worst]
    for _ in range(100):
        cases.append({k: rng.integers(0, 256, int(rng.integers(0, 120)), dtype=np.uint8).tobytes() for k in COLUMNS})
    for req in cases:
        req["duration_ms"] = -2**63
        cols, off = pack_columns([req[k] for k in COLUMNS])
        ml, dl = C.c_uint64(), C.c_uint64()
        h = np.frombuffer(b"A" * 86, dtype=np.uint8).copy()
        assert vci.hs_vci_sizes(cols.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), C.c_int64(req["duration_ms"]),
                                h.ctypes.data_as(C.c_void_p), C.byref(ml), C.byref(dl)) == 0
        bound = lib.afc_vc_issue_bound(off.ctypes.data_as(C.c_void_p), 1)
        assert bound >= dl.value and bound >= ml.value, (bound, dl.value)
    assert lib.afc_vc_issue_bound(None, 0) == 0
