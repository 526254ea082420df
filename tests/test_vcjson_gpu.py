"""Credential documents in any JSON spelling verified on the GPU (afc_vc_verify_json_batch, VCService.verify_*vc_json_batch): the device
says what the CPU build of the same walk says, the service equals the stored-document service dict for dict, host-buffer and device
calls agree (also across forced chunk boundaries), the argument and key-set errors, and a 1 M-document pretty-printed run."""
import base64
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

VALID, INVALID, HOST, UNRESOLVED, BAD = 1, 0, 2, 3, 4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def vcj(tmp_path_factory):
    from test_vcjson_hostsim import build_cpu_walk
    return build_cpu_walk(tmp_path_factory)


def _golden_keyset(ctx):
    from conftest import golden
    from agentfield_b200.identity import KeySet
    g = golden("go_cases.json")
    pk = {c["issuer"]: c["pk"] for c in g["execution_vcs"]}
    pk.update({c["issuer_did"]: c["pk"] for c in g["workflow_vcs"]})
    dids = sorted(pk)
    return KeySet([bytes.fromhex(pk[d]) for d in dids], ctx, dids=dids), set(dids)


def _signed_random_corpus(ctx, vcj, n=200):
    """Random issued documents re-spelled at random, each signed over the message the CPU build re-marshals from it (the proof is
    not part of that message, so its proofValue can be replaced afterwards).  Returns (key set, [(kind, document, message)])."""
    import re
    import test_vcjson_hostsim as H
    from agentfield_b200 import ExpandedKeys
    from agentfield_b200.identity import KeySet
    cache = ExpandedKeys(ctx)
    rng, wrng = np.random.default_rng(0xAFD0), np.random.default_rng(0xAFE0)
    own = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (8000 + a) for a in range(99)])
    names = ["did:key:z6Mk%d" % a for a in range(99)]              # the issuers the random documents name
    ks = KeySet([cache.public_key(d) for d in own], ctx, dids=names)
    out = []
    for i in range(n):
        kind = i % 2
        _, doc = (H._rand_exec if kind == 0 else H._rand_wf)(rng, rng.integers(0, 256, 64, dtype=np.uint8).tobytes())
        d = H._respell_random(wrng, H.parse_keep(doc))
        st, msg, _, sp = H.run(vcj, kind, d)
        if st != HOST:
            iss = d[sp[0]:sp[0] + sp[1]].decode()
            sig = bytes(cache.sign_batch([own[names.index(iss)]], [msg])[0])
            pv = base64.urlsafe_b64encode(sig).rstrip(b"=")
            d = re.sub(rb'("proofValue"\s*:\s*")[^"]*"', lambda m: m.group(1) + pv + b'"', d, count=1)
            out.append((kind, d, (msg, sig)))
        else:
            out.append((kind, d, None))
    return ks, out


def _golden_corpus():
    """Golden documents in every client spelling with the targeted declines, and every single-byte mutation of two pretty-printed
    golden documents: (kind, document, the reference's signing bytes and signature of the document it came from)."""
    import test_vcjson_hostsim as H
    out = []
    canon = {}
    for kind, doc, c in H._golden_docs():
        canon[doc] = (c["expect_canonical"].encode("utf-8"), bytes.fromhex(c["expect_sig"]))
        for how in H.SPELLINGS:
            s = H.spell(doc, how)
            out.append((kind, s, canon[doc]))
            if how == "indent2":
                out += [(kind, t.encode("utf-8", "surrogatepass"), canon[doc]) for _, t in H._declines(s, kind)]
    srcs = H._golden_docs()
    for (kind, src), (_, doc, _) in zip(H._indent2_sources(), (srcs[0], srcs[10])):
        for i in range(len(src)):
            out += [(kind, src[:i] + src[i + 1:], canon[doc]), (kind, src[:i + 1] + src[i:], canon[doc])]
            out += [(kind, src[:i] + b + src[i + 1:], canon[doc]) for b in H.SUBS + [b"\t", b"\n", b"\r"] if src[i:i + 1] != b]
    return out


def _compare(vcj, ks, known, corpus):
    """Device statuses and spans against the CPU build.  Each document carries a (message, signature) pair that verifies: the device
    says VALID exactly when it re-marshalled that message and decoded that signature, so where the CPU build's message and signature
    are those the device's bytes are the CPU build's, and where they are not the device must not verify."""
    import test_vcjson_hostsim as H
    counts = {VALID: 0, INVALID: 0, HOST: 0}
    for kind in (0, 1):
        docs = [(d, m) for k, d, m in corpus if k == kind]
        st, fl = ks.verify_json(kind, [d for d, _ in docs])
        for (d, signed), s, f in zip(docs, st, fl):
            cst, msg, sig, sp = H.run(vcj, kind, d)
            if cst == HOST:
                assert s == HOST, d[:200]
                counts[HOST] += 1
                continue
            assert list(f) == sp[:4], d[:200]
            if d[sp[0]:sp[0] + sp[1]].decode() not in known:
                assert s == UNRESOLVED
            elif cst == VALID:
                assert s == (VALID if (msg, sig) == signed else INVALID), (s, d[:200])
                counts[s] += 1
            else:
                assert s == cst
    return counts


def test_device_equals_cpu_build(ctx, vcj):
    """The golden corpus (client spellings, targeted declines, every single-byte mutation of two pretty-printed documents) and random
    re-spelled documents: the device's statuses and spans are the CPU build's, and its signing bytes are the CPU build's (a document
    verifies on the device exactly when the CPU build's message is the one it was signed over)."""
    ks, known = _golden_keyset(ctx)
    counts = _compare(vcj, ks, known, _golden_corpus())
    assert counts[VALID] > 1000 and counts[INVALID] > 1000 and counts[HOST] > 1000, counts
    ks.close()
    ks, corpus = _signed_random_corpus(ctx, vcj)
    counts = _compare(vcj, ks, {"did:key:z6Mk%d" % a for a in range(99)}, corpus)
    assert counts[VALID] > 150 and counts[INVALID] == 0, counts
    ks.close()


def test_negative_zero_respelled_as_zero_is_invalid(ctx):
    """A document signed over metadata holding -0, sent through plain json.loads / json.dumps (which write 0, as JSON.stringify does):
    Go re-marshals 0, not the signed -0, so the verdict is INVALID; the -0 spelling itself verifies."""
    import json
    from test_vcdoc_gpu import _service
    from test_host_logic import _vc_requests
    cache, dids, svc = _service(ctx, n_issuers=4)
    rng = np.random.default_rng(0xAFE1)
    v = svc.generate_execution_vc_batch(_vc_requests(1, dids, rng))[0]
    doc = v["doc"]
    doc["credentialSubject"]["audit"]["metadata"] = {"!": -0.0, "agentfield_version": "1.0.0"}
    from agentfield_b200 import go_json as GJ
    sig = cache.sign_batch([doc["issuer"]], [GJ.vc_document(doc)])[0]
    proof = dict(v["proof"], proofValue=base64.urlsafe_b64encode(sig).rstrip(b"=").decode())
    signed = GJ.vc_document(doc, proof)
    assert b'"!":-0,' in signed
    plain = json.dumps(json.loads(signed), indent=2).encode()
    ks = svc._named_keyset()
    st, _ = ks.verify_json(0, [signed, plain])
    assert list(st) == [VALID, INVALID]


def _mixed(ctx):
    """Issued execution and workflow documents, canonical, re-spelled and damaged (changed value, unknown issuer, undecodable
    proofValue, members swapped)."""
    import test_vcjson_hostsim as H
    from test_vcdoc_gpu import _mix, _service
    from test_host_logic import _vc_requests
    cache, dids, svc = _service(ctx)
    rng = np.random.default_rng(0xAFE2)
    issued = [v["vc_document"] for v in svc.generate_execution_vc_batch(_vc_requests(400, dids, rng, pad_to=1536))]
    wfs = [w["vc_document"] for w in svc.generate_workflow_vc_batch([
        {"workflow_id": "wf-%d" % w, "root_did": dids[w % 64], "vc_id": "v%d" % w, "workflow_vc_id": "w%d" % w,
         "issuance_date": "2026-09-21T06:00:00Z", "snapshot_time": "2026-09-21T06:00:00Z", "proof_created": "2026-09-21T06:00:01Z",
         "execution_vcs": [{"vc_id": "e%d-%d" % (w, j), "session_id": "s%d" % w, "status": ("succeeded", "failed")[j % 2],
                            "created_at": "2026-09-21T06:00:0%dZ" % j, "issuer_did": dids[w % 64]} for j in range(w % 5)]}
        for w in range(200)])]
    foreign = "did:key:z" + "Q" * 46
    out = {}
    for kind, docs in ((0, issued), (1, wfs)):
        mixed = [m for m, _ in _mix(docs, rng, foreign)]
        hows = sorted(H.SPELLINGS)
        spelled = [H.spell(m, hows[i % len(hows)]) if i % 3 else m for i, m in enumerate(mixed)]
        spelled += [H._swap_members(H.spell(m, "indent2").decode(), '"id"', '"issuer"').encode() for m in mixed[:20]]
        out[kind] = spelled
    return svc, out


def test_service_equals_stored_service(ctx):
    svc, docs = _mixed(ctx)
    for kind, verify_json, verify_stored in ((0, svc.verify_vc_json_batch, svc.verify_stored_vc_batch),
                                             (1, svc.verify_workflow_vc_json_batch, svc.verify_stored_workflow_vc_batch)):
        a, b = verify_json(docs[kind]), verify_stored(docs[kind])
        assert a == b
        st, _ = svc._named_keyset().verify_json(kind, docs[kind])
        assert (st == HOST).sum() < len(st) // 8                       # the swapped-member documents, and little else
        assert sum(r["valid"] for r in a) > len(a) // 3
        for s in (VALID, INVALID, UNRESOLVED, BAD):
            assert (st == s).any(), s


def test_host_and_device_calls_agree(ctx):
    import torch
    from agentfield_b200.crypto import pack
    svc, docs = _mixed(ctx)
    ks = svc._named_keyset()
    dev = torch.device("cuda", 0)
    for kind in (0, 1):
        buf, off = pack(docs[kind])
        st, fl = ks.verify_json_packed(kind, buf, off)
        n = len(docs[kind])
        d_st = torch.empty(n, dtype=torch.uint8, device=dev)
        d_f = torch.empty((n, 4), dtype=torch.int32, device=dev)
        ks.verify_json_dev(kind, torch.from_numpy(buf).to(dev), torch.from_numpy(off.view(np.int64)).to(dev), n, d_st, d_f)
        torch.cuda.synchronize()
        assert (st == d_st.cpu().numpy()).all() and (fl == d_f.cpu().numpy().view(np.uint32)).all()


def test_chunk_boundaries_in_a_fresh_process():
    """The host-buffer call with chunks of 97 documents (AFC_CHUNK_ITEMS is read once per process)."""
    env = dict(os.environ, AFC_CHUNK_ITEMS="97", AFC_MIN_CHUNK_ITEMS="97")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_vcjson_gpu.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "test_host_and_device_calls_agree or test_service_equals_stored_service"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "2 passed" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


def test_arguments_and_key_set_errors(ctx):
    from agentfield_b200 import _abi
    from agentfield_b200.identity import KeySet
    from oracle import c_oracle as CO
    lib, h = _abi.load(), ctx.handle
    rng = np.random.default_rng(0xAFE3)
    pks = [CO.pubkey(rng.integers(0, 256, 32, dtype=np.uint8).tobytes()) for _ in range(3)]
    plain = KeySet(pks, ctx)
    named = KeySet(pks, ctx, dids=["did:a", "did:b", "did:c"])
    doc = b"{ }"
    off = np.array([0, 3], dtype=np.uint64)
    st = np.zeros(1, dtype=np.uint8)
    f = lib.afc_vc_verify_json_batch
    assert f(h, plain.handle, 0, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_ESTATE
    assert f(h, named.handle, 0, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == 0 and st[0] == HOST
    assert f(h, named.handle, 0, None, _abi.ptr(np.zeros(1, dtype=np.uint64)), 0, None, None) == 0     # empty batch
    assert f(h, named.handle, 2, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert f(h, named.handle, -1, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert f(h, named.handle, 0, doc, None, 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert f(h, named.handle, 0, None, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert f(h, named.handle, 0, doc, _abi.ptr(off), 1, None, None) == _abi.AFC_EINVAL
    assert f(h, None, 0, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert f(None, named.handle, 0, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    back = np.array([3, 0], dtype=np.uint64)
    assert f(h, named.handle, 0, doc, _abi.ptr(back), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL        # offsets run backwards
    g = lib.afc_vc_verify_json_batch_dev
    assert g(h, named.handle, 0, None, None, 0, None, None, None) == _abi.AFC_EINVAL
    assert g(h, plain.handle, 0, None, None, 0, None, None, None) == _abi.AFC_EINVAL
    import torch
    dev = torch.device("cuda", 0)
    d_doc = torch.tensor(list(doc), dtype=torch.uint8, device=dev)
    d_off = torch.tensor([0, len(doc)], dtype=torch.int64, device=dev)
    d_st = torch.full((1,), 9, dtype=torch.uint8, device=dev)
    assert g(h, plain.handle, 0, _abi.ptr(d_doc), _abi.ptr(d_off), 1, _abi.ptr(d_st), None, None) == _abi.AFC_ESTATE   # no DIDs
    assert g(h, named.handle, 3, _abi.ptr(d_doc), _abi.ptr(d_off), 1, _abi.ptr(d_st), None, None) == _abi.AFC_EINVAL
    assert g(h, named.handle, 0, _abi.ptr(d_doc), _abi.ptr(d_off), 1, _abi.ptr(d_st), None, None) == 0
    torch.cuda.synchronize()
    assert int(d_st[0]) == HOST
    plain.close(); named.close()


def test_one_million_pretty_printed_documents(ctx):
    """2^20 execution VCs from 1024 issuers in the indent=2 spelling, 1 % with a corrupted signature: nothing goes to the host and
    every status is as planted."""
    import torch
    from agentfield_b200.respell import respelled_stored_vcs_dev
    dev = torch.device("cuda", 0)
    n = 1 << 20
    d_docs, d_off, ks, want = respelled_stored_vcs_dev(ctx, dev, n, 1024, 0xAFE4, "indent2")
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    ks.verify_json_dev(0, d_docs, d_off, n, d_st)
    torch.cuda.synchronize()
    assert int((d_st == HOST).sum()) == 0
    assert torch.equal(d_st, want)
    ks.close()
