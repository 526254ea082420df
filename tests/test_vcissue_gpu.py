"""afc_vc_issue_execution_batch[_dev] on the GPU: documents, proofValues and hashes equal oracle/ref_vc.generate_execution_vc (OpenSSL
signatures) in both signing modes; the host-buffer call equals the _dev call (also with chunks that split the batch); every issued
document verifies and audits clean against the records built from the call's outputs; with a log the root equals oracle/merkle.py and
a separate append; the argument errors; and a 2^20-credential run with every output checked."""
import base64
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MASTER = bytes(range(32))


def _keys(ctx, k, base=7000):
    import agentfield_b200 as afb
    from oracle import go_hash as H
    cache = afb.ExpandedKeys(ctx)
    paths = ["m/44'/%d'/0'" % (base + a) for a in range(k)]
    dids = cache.derive(MASTER, paths)
    seeds = {d: H.derive_seed(MASTER, p) for d, p in zip(dids, paths)}
    return cache, dids, seeds


def _varied_requests(dids, n, seed):
    """Requests with strings of every escape class (valid UTF-8: invalid bytes are covered on the CPU), error messages past 500 bytes
    cut inside runes, extreme durations, nil / empty / long payloads."""
    from agentfield_b200 import canonical as CA
    reqs = CA.synthetic_issue_requests(dids, n, seed=seed, payload_bytes=(0, 700), nil_frac=0.1, err_frac=0.2)
    rng = np.random.default_rng(seed)
    odd = ['q"uote', "back\\slash", "ctl\x00\x01\x1f\x7f", "<html>&amp;", "line\u2028sep", "para\u2029sep", "é中\U0001F600", "", "tab\there"]
    for i, r in enumerate(reqs):
        for k in ("vc_id", "execution_id", "workflow_id", "session_id", "caller_type", "target_did", "function_name", "status", "timestamp",
                  "issuance_date", "proof_created"):
            if rng.random() < 0.08:
                r[k] = r[k] + odd[int(rng.integers(len(odd)))]
        if i % 50 == 3:
            r["duration_ms"] = int(rng.choice([-1, -2**63, 2**63 - 1, 0, -123456789012345678]))
        if i % 37 == 5:
            r["error_message"] = "x" * int(rng.integers(497, 503)) + "é✓\U0001D11E" * 3
        if i % 41 == 6:
            r["input"] = b""
    return reqs


def _oracle(reqs, seeds):
    from oracle import go_hash as H, ref_vc as RV
    out = []
    for r in reqs:
        rr = dict(r)
        for k in ("input", "output"):
            rr[k] = None if r[k] is None else bytes(r[k])
        o = RV.generate_execution_vc(rr, seeds[r["caller_did"]])
        out.append((o["vc_document"], o["signature"], H.hash_data(H.marshal_data_or_null(rr["input"])),
                    H.hash_data(H.marshal_data_or_null(rr["output"]))))
    return out


def _dev_issue(ctx, cache, reqs, hash_data=True, log=None):
    import torch
    dev = torch.device("cuda", ctx.device)
    cols, coff, dur, pay, poff, nil = cache.pack_issue_requests(reqs)
    t = lambda a: torch.from_numpy(a).to(dev)
    ki = cache.key_index([r["caller_did"] for r in reqs])
    d_docs, d_off, d_h, d_pv = cache.issue_dev(t(ki.view(np.int32)), t(cols), t(coff.view(np.int64)), t(dur), t(pay), t(poff.view(np.int64)), t(nil),
                                               len(reqs), hash_data=hash_data, log=log)
    torch.cuda.synchronize(dev)
    return (d_docs.cpu().numpy().tobytes(), d_off.cpu().numpy().astype(np.uint64), None if d_h is None else d_h.cpu().numpy(), d_pv.cpu().numpy())


def _host_issue(cache, reqs, hash_data=True, log=None):
    ki = cache.key_index([r["caller_did"] for r in reqs])
    docs, off, h, pv = cache.issue_packed(ki, *cache.pack_issue_requests(reqs), hash_data=hash_data, log=log)
    return docs.tobytes(), off, h, pv


def _split(res, n):
    docs, off, h, pv = res
    return [(docs[int(off[i]):int(off[i + 1])], pv[i].tobytes().decode(), "" if h is None else h[i, :43].tobytes().decode(),
             "" if h is None else h[i, 43:].tobytes().decode()) for i in range(n)]


@pytest.mark.parametrize("constant_time", [True, False])
def test_equals_oracle(ctx, constant_time):
    cache, dids, seeds = _keys(ctx, 24)
    reqs = _varied_requests(dids, 2000, seed=11)
    want = _oracle(reqs, seeds)
    ctx.sign_configure(constant_time)
    try:
        got_dev = _split(_dev_issue(ctx, cache, reqs), len(reqs))
        got_host = _split(_host_issue(cache, reqs), len(reqs))
    finally:
        ctx.sign_configure(True)
    for i, (w, d, h) in enumerate(zip(want, got_dev, got_host)):
        assert d == w, (i, d, w)
        assert h == w, i


def test_hash_data_off_and_empty_batch(ctx):
    from oracle import go_ed25519 as G, ref_vc as RV
    cache, dids, seeds = _keys(ctx, 4)
    reqs = _varied_requests(dids, 300, seed=12)
    got = _split(_host_issue(cache, reqs, hash_data=False), len(reqs))
    assert got == _split(_dev_issue(ctx, cache, reqs, hash_data=False), len(reqs))
    for r, g in zip(reqs, got):
        assert g[2] == g[3] == ""
        canonical = RV.go_marshal(RV.vc_document(r, "", ""))
        proof = {"type": "Ed25519Signature2020", "created": r["proof_created"], "verificationMethod": "%s#key-1" % r["caller_did"],
                 "proofPurpose": "assertionMethod", "proofValue": g[1]}
        assert g[0] == RV.go_marshal(RV.vc_document(r, "", "", proof))
        assert G.verify(cache.public_key(r["caller_did"]), canonical, base64.urlsafe_b64decode(g[1] + "=="))
    docs, off, h, pv = _host_issue(cache, [])
    assert off.tolist() == [0] and pv.shape == (0, 86)


def test_service_is_one_call_and_unchanged(ctx):
    """VCService(canonical_on_device=True) returns exactly what the host path returns."""
    from agentfield_b200.services import VCService
    cache, dids, _ = _keys(ctx, 8)
    reqs = _varied_requests(dids, 400, seed=13)
    a = VCService(cache, canonical_on_device=True).generate_execution_vc_batch(reqs)
    b = VCService(cache, canonical_on_device=False).generate_execution_vc_batch(reqs)
    assert a == b
    before = ctx.launch_count()
    VCService(cache, canonical_on_device=True, hash_sensitive_data=False).generate_execution_vc_batch(reqs[:10])
    assert ctx.launch_count() - before < 20


def test_issued_documents_verify_and_audit_clean(ctx):
    from agentfield_b200 import _abi
    from agentfield_b200.identity import KeySet
    from agentfield_b200.services import normalize_execution_status
    cache, dids, _ = _keys(ctx, 16)
    reqs = _varied_requests(dids, 1500, seed=14)
    for r in reqs:
        # what the stored-document verifier proves canonical itself (it leaves durations past 2^53 and the U+FFFD of a message cut
        # inside a rune to the host), with the RFC 3339 date and printable status the audit's rules decide on the device
        r["issuance_date"] = "2026-09-21T06:00:00Z"
        r["status"] = "succeeded"
        r["duration_ms"] = abs(r["duration_ms"]) % 10 ** 9
        if len(r["error_message"].encode()) > 500:
            r["error_message"] = r["error_message"][:120]
    got = _split(_dev_issue(ctx, cache, reqs), len(reqs))
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    st, _ = ks.verify_stored(_abi.DOC_EXECUTION_VC, [g[0] for g in got])
    assert (st == _abi.VC_VALID).all()
    cols = [[r["caller_did"], r["execution_id"], r["workflow_id"], r["session_id"], r["caller_did"], r["target_did"],
             normalize_execution_status(r["status"]), g[2], g[3], g[1]] for r, g in zip(reqs, got)]
    st, iss = ks.audit_stored(_abi.DOC_EXECUTION_VC, [g[0] for g in got], cols)
    assert (st == _abi.VC_VALID).all() and (iss == 0).all()
    ks.close()


def test_log_root(ctx):
    import agentfield_b200 as afb
    from oracle import merkle as OM
    cache, dids, _ = _keys(ctx, 8)
    reqs = _varied_requests(dids, 700, seed=15)
    log_dev, log_host, ref = afb.Auditor(ctx), afb.Auditor(ctx), afb.Auditor(ctx)
    d = _split(_dev_issue(ctx, cache, reqs[:300], log=log_dev), 300) + _split(_dev_issue(ctx, cache, reqs[300:], log=log_dev), 400)
    h = _split(_host_issue(cache, reqs, log=log_host), 700)
    docs = [x[0] for x in d]
    assert docs == [x[0] for x in h]
    root, size = ref.append(docs)
    assert size == 700 and log_dev.root() == log_host.root() == (root, 700)
    assert root == OM.root(docs)


def test_host_and_device_calls_agree(ctx):
    cache, dids, _ = _keys(ctx, 32)
    reqs = _varied_requests(dids, 1000, seed=16)
    assert _split(_host_issue(cache, reqs), 1000) == _split(_dev_issue(ctx, cache, reqs), 1000)


def test_chunk_boundaries_in_a_fresh_process():
    """The host-buffer calls with chunks of 97 requests (AFC_CHUNK_ITEMS is read once per process)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, AFC_CHUNK_ITEMS="97", AFC_MIN_CHUNK_ITEMS="97")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(root, "tests", "test_vcissue_gpu.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "test_host_and_device_calls_agree or test_log_root"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "2 passed" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


def test_argument_errors(ctx):
    import ctypes as C
    import torch
    import agentfield_b200 as afb
    from agentfield_b200 import _abi
    lib = _abi.load()
    cache, dids, _ = _keys(ctx, 2)
    reqs = _varied_requests(dids, 5, seed=17)
    ki = cache.key_index([r["caller_did"] for r in reqs])
    cols, coff, dur, pay, poff, nil = cache.pack_issue_requests(reqs)
    exp = cache._expanded
    cap = lib.afc_vc_issue_bound(_abi.ptr(coff), 5)
    docs, doff = np.empty(cap, dtype=np.uint8), np.zeros(6, dtype=np.uint64)
    h, pv = np.empty((5, 86), dtype=np.uint8), np.empty((5, 86), dtype=np.uint8)
    P = _abi.ptr

    def call(**kw):
        a = dict(exp=exp, nk=exp.shape[0], ki=ki, cols=cols, coff=coff, dur=dur, pay=pay, poff=poff, nil=nil, flags=_abi.ISSUE_HASH_DATA,
                 log=None, docs=docs, cap=cap, doff=doff, h=h, pv=pv)
        a.update(kw)
        return lib.afc_vc_issue_execution_batch(ctx.handle, P(a["exp"]), a["nk"], P(a["ki"]), P(a["cols"]), P(a["coff"]), P(a["dur"]), P(a["pay"]),
                                                P(a["poff"]), P(a["nil"]), a["flags"], 5, a["log"], P(a["docs"]), a["cap"], P(a["doff"]), P(a["h"]),
                                                P(a["pv"]))
    assert call() == _abi.AFC_OK
    assert call(cap=cap - 1) == _abi.AFC_EINVAL
    bad = ki.copy(); bad[3] = exp.shape[0]
    assert call(ki=bad) == _abi.AFC_EINVAL
    assert call(h=None) == _abi.AFC_EINVAL
    assert call(h=None, flags=0) == _abi.AFC_OK
    assert call(flags=2) == _abi.AFC_EINVAL
    assert call(nk=0) == _abi.AFC_EINVAL
    for k in ("exp", "ki", "cols", "coff", "dur", "pay", "poff", "nil", "docs", "doff", "pv"):
        assert call(**{k: None}) == _abi.AFC_EINVAL, k
    back = coff.copy(); back[20] = back[19] - 1
    assert call(coff=back) == _abi.AFC_EINVAL
    pback = poff.copy(); pback[4] = pback[3] - 1 if pback[3] else 0; pback[3] = pback[3] + 5
    assert call(poff=pback) == _abi.AFC_EINVAL
    other = afb.Context(0)
    foreign = afb.Auditor(other)
    assert call(log=foreign.handle) == _abi.AFC_EINVAL
    assert lib.afc_vc_issue_execution_batch(None, P(exp), 1, P(ki), P(cols), P(coff), P(dur), P(pay), P(poff), P(nil), 0, 5, None, P(docs), cap,
                                            P(doff), P(h), P(pv)) == _abi.AFC_EINVAL
    # the _dev call: too small a buffer, hashes missing with HASH_DATA
    dev = torch.device("cuda", ctx.device)
    t = lambda a: torch.from_numpy(a).to(dev)
    d = dict(exp=t(exp), ki=t(ki.view(np.int32)), cols=t(cols), coff=t(coff.view(np.int64)), dur=t(dur), pay=t(pay), poff=t(poff.view(np.int64)),
             nil=t(nil), docs=torch.empty(cap, dtype=torch.uint8, device=dev), doff=torch.empty(6, dtype=torch.int64, device=dev),
             h=torch.empty((5, 86), dtype=torch.uint8, device=dev), pv=torch.empty((5, 86), dtype=torch.uint8, device=dev))

    def dcall(cap_, h_):
        return lib.afc_vc_issue_execution_batch_dev(ctx.handle, P(d["exp"]), exp.shape[0], P(d["ki"]), P(d["cols"]), P(d["coff"]), P(d["dur"]),
                                                    P(d["pay"]), P(d["poff"]), P(d["nil"]), _abi.ISSUE_HASH_DATA, 5, None, P(d["docs"]), cap_,
                                                    P(d["doff"]), h_, P(d["pv"]), ctx._stream(None))
    assert dcall(cap, P(d["h"])) == _abi.AFC_OK
    assert dcall(cap - 1, P(d["h"])) == _abi.AFC_EINVAL
    assert dcall(cap, None) == _abi.AFC_EINVAL
    torch.cuda.synchronize(dev)
    foreign.close(); other.close()


def _fast_expected(r, ih, oh, pv):
    """json.Marshal of the stored document for requests whose strings need no escaping and carry no error message."""
    did, agent = r["caller_did"], r["agent_node_did"]
    return ('{"@context":["https://www.w3.org/2018/credentials/v1","https://agentfield.example.com/contexts/execution/v1"],'
            '"type":["VerifiableCredential","AgentFieldExecutionCredential"],"id":"urn:agentfield:vc:%s","issuer":"%s","issuanceDate":"%s",'
            '"credentialSubject":{"executionId":"%s","workflowId":"%s","sessionId":"%s","caller":{"did":"%s","type":"%s","agentNodeDid":"%s"},'
            '"target":{"did":"%s","agentNodeDid":"%s","functionName":"%s"},"execution":{"inputHash":"%s","outputHash":"%s","timestamp":"%s",'
            '"durationMs":%d,"status":"%s"},"audit":{"inputDataHash":"%s","outputDataHash":"%s",'
            '"metadata":{"agentfield_version":"1.0.0","vc_version":"1.0"}}},"proof":{"type":"Ed25519Signature2020","created":"%s",'
            '"verificationMethod":"%s#key-1","proofPurpose":"assertionMethod","proofValue":"%s"}}'
            % (r["vc_id"], did, r["issuance_date"], r["execution_id"], r["workflow_id"], r["session_id"], did, r["caller_type"], agent,
               r["target_did"], agent, r["function_name"], ih, oh, r["timestamp"], r["duration_ms"], r["status"], ih, oh, r["proof_created"], did,
               pv)).encode()


def test_one_million_credentials(ctx):
    """2^20 requests from 1024 issuers: every hash equals hashlib's, every document equals its expected bytes (built from the request
    and the returned hashes and proofValue; the mirror for the ~1 % with an error message), and every document verifies."""
    import torch
    from agentfield_b200 import _abi, go_json
    from agentfield_b200.identity import KeySet
    n = 1 << 20
    cache, dids, _ = _keys(ctx, 1024, base=9000)
    from agentfield_b200 import canonical as CA
    reqs = CA.synthetic_issue_requests(dids, n, seed=18, payload_bytes=(0, 512))
    docs, off, h, pv = _dev_issue(ctx, cache, reqs)
    bad = 0
    for i, r in enumerate(reqs):
        ih, oh = h[i, :43].tobytes().decode(), h[i, 43:].tobytes().decode()
        for k, d in ((0, r["input"]), (1, r["output"])):
            m = b"null" if d is None else b'"' + base64.b64encode(d) + b'"'
            bad += (ih, oh)[k] != base64.urlsafe_b64encode(hashlib.sha256(m).digest()).rstrip(b"=").decode()
        p = pv[i].tobytes().decode()
        doc = docs[int(off[i]):int(off[i + 1])]
        if r["error_message"]:
            em = go_json.truncate_error_message(r["error_message"])
            d = {"@context": ["https://www.w3.org/2018/credentials/v1", "https://agentfield.example.com/contexts/execution/v1"],
                 "type": ["VerifiableCredential", "AgentFieldExecutionCredential"], "id": "urn:agentfield:vc:%s" % r["vc_id"], "issuer": r["caller_did"],
                 "issuanceDate": r["issuance_date"],
                 "credentialSubject": {"executionId": r["execution_id"], "workflowId": r["workflow_id"], "sessionId": r["session_id"],
                                       "caller": {"did": r["caller_did"], "type": r["caller_type"], "agentNodeDid": r["agent_node_did"]},
                                       "target": {"did": r["target_did"], "agentNodeDid": r["agent_node_did"], "functionName": r["function_name"]},
                                       "execution": {"inputHash": ih, "outputHash": oh, "timestamp": r["timestamp"], "durationMs": r["duration_ms"],
                                                     "status": r["status"], "errorMessage": em},
                                       "audit": {"inputDataHash": ih, "outputDataHash": oh,
                                                 "metadata": {"agentfield_version": "1.0.0", "vc_version": "1.0"}}}}
            proof = {"type": "Ed25519Signature2020", "created": r["proof_created"], "verificationMethod": "%s#key-1" % r["caller_did"],
                     "proofPurpose": "assertionMethod", "proofValue": p}
            bad += doc != go_json.vc_document(d, proof)
        else:
            bad += doc != _fast_expected(r, ih, oh, p)
    assert bad == 0 and int(off[n]) == len(docs)
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    dev = torch.device("cuda", ctx.device)
    d_docs = torch.from_numpy(np.frombuffer(docs, dtype=np.uint8).copy()).to(dev)
    d_off = torch.from_numpy(off.view(np.int64)).to(dev)
    st = torch.empty(n, dtype=torch.uint8, device=dev)
    ks.verify_stored_dev(_abi.DOC_EXECUTION_VC, d_docs, d_off, n, st)
    torch.cuda.synchronize(dev)
    assert (st.cpu().numpy() == _abi.VC_VALID).all()
    ks.close()
