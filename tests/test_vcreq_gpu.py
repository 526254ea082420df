"""VC verification requests answered on the GPU (afc_vc_verify_request_batch, KeySet.verify_requests*, VCService.serve_verify_requests):
byte-for-byte parity with the CPU build of the same logic and with the oracle on a corpus of more than 10 000 request bodies covering every
response row, the host-buffer and device calls agree (also across forced chunk boundaries), the statuses agree with
afc_vc_verify_json_batch on the same documents, every argument error and n = 0, 2^20 requests with nothing left to the host, and the
service equals the oracle for every request, the ones the device leaves to the host included."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import test_vcreq_hostsim as H
import verify_request_oracle as O
from conftest import golden

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, ESTATE = -1, -5


@pytest.fixture(scope="module")
def vrq(tmp_path_factory):
    return H.build_cpu_request(tmp_path_factory)


def _keyset(ctx):
    from agentfield_b200.identity import KeySet
    reg = H.registry()
    dids = sorted(reg)
    return KeySet([reg[d] for d in dids], ctx, dids=dids), reg


def _variants(doc_bytes):
    """One document with each verdict: as issued, an unknown issuer, a bad base64 character, a base64 length of 1 mod 4, a wrong signature,
    an issuance date that needs escaping."""
    d = json.loads(doc_bytes)
    pv = d["proof"]["proofValue"]
    out = []
    for iss, p, date in ((d["issuer"], pv, d["issuanceDate"]), ("did:key:z6MkUnknown<&> ", pv, d["issuanceDate"]),
                         (d["issuer"], pv[:20] + "=" + pv[21:], d["issuanceDate"]), (d["issuer"], pv + "AAA", d["issuanceDate"]),
                         (d["issuer"], pv[:-2] + ("B" if pv[-2] != "B" else "C") + pv[-1], d["issuanceDate"]),
                         (d["issuer"], pv, d["issuanceDate"] + " <é >"), ("", pv, "")):
        out.append(json.dumps(dict(d, issuer=iss, issuanceDate=date, proof=dict(d["proof"], proofValue=p))).encode())
    return out


def corpus():
    """More than 10 000 request bodies: every shape of every realistic document and its verdict variants, the envelopes of the CPU test,
    non-object values, every truncation of one body and every single-byte deletion and substitution of another."""
    docs = H.realistic_docs()
    bodies = []
    for doc in docs:
        bodies += [shape(doc) for shape in H.SHAPES]
        for v in _variants(doc):
            bodies += [b'{"vc_document":' + v + b'}', H.ui_body(v), H.pretty_body(v)]
    doc = docs[2]
    bodies += [b'{"a":1,"vc_document":' + doc + b',"z":[{}]}', b'{"VC_DOCUMENT":' + doc + b'}', b'{"vc_document":' + doc + b'} x',
               b'{"vc_document":' + docs[3] + b',"vc_document":' + doc + b'}', b'{"vc_document":' + doc + b',"vc_document":null}',
               b'\xef\xbb\xbf{}', b'', b' ', b'[]', b'"x"', b'1', b'true', b'false', b'null', b'{}', b'{"vc_document":null}',
               b'{"vc_document":"x"}', b'{"vc_document":[]}', b'{"vc_document":-1e5}', b'{"vc_document":false}', b'{"vc_document":{}}',
               b'{"vc_\\u0064ocument":' + doc + b'}', b'{"a":' + b"[" * 80 + b"]" * 80 + b'}', b'{"x":"\\ud800"}', b'{"x":1.5e+3}']
    body = H.sdk_body(docs[0])
    bodies += [body[:i] for i in range(len(body))]
    body = H.ui_body(docs[1])
    for i in range(len(body)):
        bodies += [body[:i] + body[i + 1:]] + [body[:i] + s + body[i + 1:] for s in H.SUBS if body[i:i + 1] != s]
    return bodies


@pytest.fixture(scope="module")
def setup(ctx, vrq):
    ks, reg = _keyset(ctx)
    bodies = corpus()
    assert len(bodies) > 10000
    res = ks.verify_requests(bodies)
    return ks, reg, bodies, res


def test_parity_with_cpu_build_and_oracle(vrq, setup):
    ks, reg, bodies, res = setup
    seen = set()
    for body, got in zip(bodies, res):
        assert got == H.cpu_answer(vrq, body, reg), body[:200]
        if got[0] == O.HOST:
            assert got[1] == b""
            continue
        assert got == O.answer(body, reg), (got, body[:200])
        seen.add(got[1][:40] if got[0] == O.OK else got[1])
    rows = [b'{"valid":true', b'{"valid":false,"message":"Invalid signature"}', b'{"error":"Invalid request body"}',
            b'{"valid":false,"error":"failed to parse VC document:', b'{"valid":false,"error":"failed to resolve issuer DID:',
            b'{"valid":false,"error":"failed to verify signature:']
    for r in rows:
        assert any(s.startswith(r[:40]) for s in seen), r
    assert sum(1 for st, _ in res if st == O.HOST) < len(res) // 4


def test_host_and_device_calls_agree(setup):
    import torch
    from agentfield_b200.crypto import pack
    ks, reg, bodies, res = setup
    buf, off = pack(bodies)
    # a batch that starts past byte 0 of the request buffer
    d_reqs = torch.cat([torch.zeros(5, dtype=torch.uint8), torch.from_numpy(buf.copy())]).cuda()
    d_off = torch.from_numpy(off.astype(np.int64) + 5).cuda()
    d_bodies, d_body_off, d_state = ks.verify_requests_dev(d_reqs, d_off, len(bodies))
    torch.cuda.synchronize()
    out = d_bodies.cpu().numpy().tobytes()
    bo = d_body_off.cpu().numpy()
    st = d_state.cpu().numpy()
    assert [(int(st[i]), out[bo[i]:bo[i + 1]]) for i in range(len(bodies))] == res


def test_chunk_boundaries_in_a_fresh_process(setup, tmp_path):
    ks, reg, bodies, res = setup
    sample = bodies[:600] + bodies[-600:]
    want = res[:600] + res[-600:]
    inp, outp = tmp_path / "in.json", tmp_path / "out.json"
    inp.write_text(json.dumps({"bodies": [b.hex() for b in sample], "reg": {d: pk.hex() for d, pk in reg.items()}}))
    code = ("import json, sys\n"
            "sys.path.insert(0, %r)\n"
            "import agentfield_b200 as afb\n"
            "from agentfield_b200.identity import KeySet\n"
            "a = json.load(open(%r))\n"
            "ctx = afb.Context(0)\n"
            "dids = sorted(a['reg'])\n"
            "ks = KeySet([bytes.fromhex(a['reg'][d]) for d in dids], ctx, dids=dids)\n"
            "r = ks.verify_requests([bytes.fromhex(b) for b in a['bodies']])\n"
            "json.dump([[s, b.hex()] for s, b in r], open(%r, 'w'))\n"
            "ks.close(); ctx.close()\n") % (ROOT, str(inp), str(outp))
    env = dict(os.environ, AFC_CHUNK_ITEMS="7", AFC_MIN_CHUNK_ITEMS="3")
    subprocess.check_call([sys.executable, "-c", code], env=env, timeout=600)
    got = [(s, bytes.fromhex(b)) for s, b in json.load(open(outp))]
    assert got == want


def test_statuses_agree_with_json_verify(vrq, setup):
    import ctypes as C
    ks, reg, bodies, res = setup
    docs, idx = [], []
    for i, body in enumerate(bodies):
        span = (C.c_uint32 * 2)()
        if vrq.hs_vrq_bind(body, C.c_uint64(len(body)), span) == H.VRB_OBJECT:
            docs.append(body[span[0]:span[0] + span[1]])
            idx.append(i)
    status, _ = ks.verify_json(0, docs)
    prefix = {H.VC_VALID: b'{"valid":true', H.VC_INVALID: b'{"valid":false,"message":"Invalid signature"}',
              H.VC_UNRESOLVED: b'{"valid":false,"error":"failed to resolve', H.VC_BAD_ENCODING: b'{"valid":false,"error":"failed to verify'}
    for i, s in zip(idx, status):
        st, body = res[i]
        if s == H.VC_HOST:
            assert st == O.HOST
        else:
            assert st == O.OK and body.startswith(prefix[int(s)]), (s, body)


def test_argument_errors_and_empty_batches(ctx, setup):
    import torch
    import agentfield_b200 as afb
    from agentfield_b200 import _abi
    from agentfield_b200.identity import KeySet
    ks, reg, bodies, res = setup
    lib = _abi.load()
    p = _abi.ptr
    reqs = np.frombuffer(b'{"vc_document":null}' * 2, dtype=np.uint8).copy()
    off = np.array([0, 20, 40], dtype=np.uint64)
    cap = lib.afc_vc_verify_request_bound(p(off), 2)
    assert cap == 2 * lib.afc_vc_verify_request_bound(p(np.zeros(2, dtype=np.uint64)), 1) + 6 * 40
    out, bo, st = np.zeros(cap, dtype=np.uint8), np.zeros(3, dtype=np.uint64), np.zeros(2, dtype=np.uint8)
    call = lambda c, k, r, o, n, b, cp, bo_, s: lib.afc_vc_verify_request_batch(c, k, p(r), p(o), n, p(b), cp, p(bo_), p(s))   # noqa: E731
    assert call(ctx.handle, ks.handle, reqs, off, 2, out, cap, bo, st) == 0
    assert call(ctx.handle, ks.handle, reqs, off, 2, out, cap - 1, bo, st) == EINVAL
    for args in ((None, ks.handle), (ctx.handle, None)):
        assert lib.afc_vc_verify_request_batch(args[0], args[1], p(reqs), p(off), 2, p(out), cap, p(bo), p(st)) == EINVAL
    assert lib.afc_vc_verify_request_batch(ctx.handle, ks.handle, None, p(off), 2, p(out), cap, p(bo), p(st)) == EINVAL
    assert lib.afc_vc_verify_request_batch(ctx.handle, ks.handle, p(reqs), None, 2, p(out), cap, p(bo), p(st)) == EINVAL
    assert lib.afc_vc_verify_request_batch(ctx.handle, ks.handle, p(reqs), p(off), 2, None, cap, p(bo), p(st)) == EINVAL
    assert lib.afc_vc_verify_request_batch(ctx.handle, ks.handle, p(reqs), p(off), 2, p(out), cap, None, p(st)) == EINVAL
    assert lib.afc_vc_verify_request_batch(ctx.handle, ks.handle, p(reqs), p(off), 2, p(out), cap, p(bo), None) == EINVAL
    back = np.array([0, 30, 20], dtype=np.uint64)
    assert call(ctx.handle, ks.handle, reqs, back, 2, out, 1 << 20, bo, st) == EINVAL
    huge = np.array([0, 1 << 31], dtype=np.uint64)
    assert call(ctx.handle, ks.handle, reqs, huge, 1, out, 1 << 40, bo, st) == EINVAL
    # a key set without DIDs, and one of another context
    plain = KeySet([next(iter(reg.values()))], ctx)
    assert call(ctx.handle, plain.handle, reqs, off, 2, out, cap, bo, st) == ESTATE
    plain.close()
    other = afb.Context(0)
    oks = KeySet([reg[d] for d in sorted(reg)], other, dids=sorted(reg))
    assert call(ctx.handle, oks.handle, reqs, off, 2, out, cap, bo, st) == EINVAL
    oks.close()
    other.close()
    # n = 0: body_off[0] = 0 in the host call, nothing written by the device call
    bo0 = np.full(1, 77, dtype=np.uint64)
    assert call(ctx.handle, ks.handle, reqs, off, 0, out, 0, bo0, st) == 0 and bo0[0] == 0
    assert lib.afc_vc_verify_request_bound(p(off), 0) == 0
    d_bo = torch.full((1,), 77, dtype=torch.int64, device="cuda")
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    d_reqs = torch.from_numpy(reqs).cuda()
    d_out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    d_st = torch.zeros(2, dtype=torch.uint8, device="cuda")
    dev = lambda o, n, cp: lib.afc_vc_verify_request_batch_dev(ctx.handle, ks.handle, p(d_reqs), p(o), n, p(d_out), cp, p(d_bo), p(d_st),  # noqa: E731
                                                               ctx._stream(None))
    assert dev(d_off, 0, 0) == 0 and int(d_bo[0]) == 77
    d_bo = torch.zeros(3, dtype=torch.int64, device="cuda")
    assert dev(d_off, 2, cap - 1) == EINVAL
    assert dev(d_off, 2, cap) == 0
    torch.cuda.synchronize()
    assert d_st.cpu().tolist() == [O.OK, O.OK]
    assert dev(torch.tensor([0, 30, 20], dtype=torch.int64, device="cuda"), 2, 1 << 20) == EINVAL
    assert dev(torch.tensor([0, 1 << 31], dtype=torch.int64, device="cuda"), 1, 1 << 40) == EINVAL


def test_a_million_requests_none_left_to_the_host(setup):
    import torch
    ks, reg, bodies, res = setup
    distinct = []
    for doc in H.realistic_docs():
        distinct += [H.sdk_body(doc), H.ui_body(doc)] + [H.ui_body(v) for v in _variants(doc)]
    want = ks.verify_requests(distinct)
    assert all(st == O.OK for st, _ in want)
    n, k = 1 << 20, len(distinct)
    # request i is distinct[i % k]: the buffer is the distinct bodies repeated, built on the host (about 2 GB) and copied once
    full, rem = divmod(n, k)
    lens = np.array([len(b) for b in distinct], dtype=np.int64)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.concatenate([np.tile(lens, full), lens[:rem]]), out=off[1:])
    host = np.frombuffer(b"".join(distinct) * full + b"".join(distinct[:rem]), dtype=np.uint8)
    try:
        d_reqs = torch.from_numpy(host.copy()).cuda()
        del host
        d_off = torch.from_numpy(off).cuda()
        d_bodies, d_body_off, d_state = ks.verify_requests_dev(d_reqs, d_off, n)
        torch.cuda.synchronize()
        st = d_state.cpu().numpy()
        assert int((st == O.HOST).sum()) == 0 and int((st != O.OK).sum()) == 0
        bo = d_body_off.cpu().numpy()
        out = d_bodies.cpu().numpy()
        for i in list(range(0, n, 9973)) + [n - 1]:
            assert out[bo[i]:bo[i + 1]].tobytes() == want[i % k][1]
    finally:
        d_reqs = d_off = d_bodies = d_body_off = d_state = None
        torch.cuda.empty_cache()          # the tests after this one start processes of their own on the same device


def test_service_equals_oracle_for_every_request(ctx, setup):
    from agentfield_b200 import ExpandedKeys
    from agentfield_b200.services import VCService
    ks, reg, bodies, res = setup
    g = golden("go_cases.json")["execution_vcs"]
    cache = ExpandedKeys(ctx)
    seeds = np.stack([np.frombuffer(bytes.fromhex(c["seed"]), dtype=np.uint8) for c in g])
    cache._append(ctx.expand(seeds), [c["issuer"] for c in g])
    for c in g:
        assert cache.public_key(c["issuer"]) == bytes.fromhex(c["pk"])
    svc = VCService(cache, ctx)
    # the device's answers, the ones it leaves to the host, and a few more of those: an escaped member name, the empty DID, deep nesting
    doc = H.realistic_docs()[0]
    sample = bodies[:400] + [b for b, (st, _) in zip(bodies, res) if st == O.HOST][:300] + \
        [b'{"vc_\\u0064ocument":' + doc + b'}', b'{"\\u00e9":1,"vc_document":' + doc + b'}', b'{"vc_document":"x"}', b'{"vc_document":[1]}',
         b'{"vc_document":2}', b'{"vc_document":true}']
    got = svc.serve_verify_requests(sample)
    for body, (code, out) in zip(sample, got):
        want = O.answer(body, reg)
        if want is None:
            continue
        assert (code, out) == (200 if want[0] == O.OK else 400, want[1]), (code, out, want, body[:200])
