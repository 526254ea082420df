"""Stored credential documents verified on the GPU (afc_vc_verify_stored_batch, VCService.verify_stored_*_batch): every verdict equals
the host path (Unmarshal -> Marshal with a zero proof -> verify) and the oracle's signature check, host-buffer and device calls
agree (also across forced chunk boundaries), the argument and key-set errors, and a 1 M-document run."""
import base64
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from oracle import c_oracle as CO

pytestmark = pytest.mark.gpu

VALID, INVALID, HOST, UNRESOLVED, BAD = 1, 0, 2, 3, 4


def _service(ctx, n_issuers=64, seed=0xAFD5):
    from agentfield_b200 import ExpandedKeys
    from agentfield_b200.services import VCService
    rng = np.random.default_rng(seed)
    cache = ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (3000 + a) for a in range(n_issuers)])
    return cache, dids, VCService(cache, ctx)


def _expected(svc, kind, raw):
    """The reference's verdict for one stored document, computed on the host with the oracle verifying the signature."""
    from agentfield_b200 import go_json as GJ
    from agentfield_b200.services import go_unmarshal_vc
    try:
        d = go_unmarshal_vc(raw, kind)
    except ValueError:
        return "parse"
    if d["issuer"] not in svc.keys._index:
        return UNRESOLVED
    pv = d["proof"]["proofValue"]
    if not re.fullmatch(r"[A-Za-z0-9_-]*", pv) or len(pv) % 4 == 1:
        return BAD
    sig = base64.urlsafe_b64decode(pv + "=" * (-len(pv) % 4))
    if len(sig) != 64:
        return INVALID
    msg = (GJ.vc_document if kind == 0 else GJ.workflow_vc_document)(d)
    pk = np.frombuffer(svc.keys.public_key(d["issuer"]), dtype=np.uint8).reshape(1, 32)
    ok = CO.ed25519_verify_batch(pk, np.frombuffer(sig, dtype=np.uint8).reshape(1, 64), np.frombuffer(msg, dtype=np.uint8),
                                 np.array([0, len(msg)], dtype=np.uint64))
    return VALID if ok[0] else INVALID


def _mix(docs, rng, foreign_did):
    """The issued documents plus, for a share of them, each kind of damage: (document, what the device must say or None = either)."""
    out = []
    for i, d in enumerate(docs):
        k = i % 10
        s = d.decode("utf-8")
        pv = re.search(r'"proofValue":"([^"]*)"', s).group(1)
        if k == 1:                                            # corrupted signature, still base64url of 64 bytes
            j = 5 + i % 70
            s = s.replace(pv, pv[:j] + ("A" if pv[j] != "A" else "B") + pv[j + 1:])
            out.append((s.encode(), INVALID))
        elif k == 2:                                          # tampered value, still canonical
            out.append((s.replace('"issuanceDate":"2', '"issuanceDate":"3', 1).encode(), INVALID))
        elif k == 3:                                          # non-canonical rewrite Go still verifies
            out.append(((" " if i % 20 == 3 else "") + s.replace('"id":', '"id" :', 1) + "\n", HOST))
        elif k == 4:                                          # unknown issuer
            iss = re.search(r'"issuer":"([^"]*)"', s).group(1)
            out.append((s.replace('"issuer":"%s"' % iss, '"issuer":"%s"' % foreign_did, 1).encode(), UNRESOLVED))
        elif k == 5:                                          # undecodable proofValue
            out.append((s.replace(pv, pv[:7] + "+" + pv[8:]).encode(), BAD))
        else:
            out.append((d, None))
    return [(m if isinstance(m, bytes) else m.encode(), w) for m, w in out]


def test_stored_verdicts_equal_host_path_and_oracle(ctx):
    from test_host_logic import _vc_requests
    from agentfield_b200 import _abi
    from agentfield_b200.services import VCService
    cache, dids, svc = _service(ctx)
    rng = np.random.default_rng(0xAFD6)
    reqs = _vc_requests(2000, dids, rng, pad_to=1536)
    issued = svc.generate_execution_vc_batch(reqs[:1000]) + VCService(cache, ctx, canonical_on_device=True).generate_execution_vc_batch(reqs[1000:])
    wfs = svc.generate_workflow_vc_batch([{"workflow_id": "wf-%d" % w, "root_did": dids[w % 64], "vc_id": "v%d" % w, "workflow_vc_id": "w%d" % w,
                                           "issuance_date": "2026-09-21T06:00:00Z", "snapshot_time": "2026-09-21T06:00:00Z",
                                           "proof_created": "2026-09-21T06:00:01Z",
                                           "execution_vcs": [{"vc_id": "e%d-%d" % (w, j), "session_id": "s%d" % w, "status": ("succeeded", "failed")[j % 2],
                                                              "created_at": "2026-09-21T06:00:0%dZ" % j, "issuer_did": dids[w % 64]} for j in range(w % 5)]}
                                          for w in range(300)])
    foreign = "did:key:z" + "Q" * 46
    for kind, docs, verify in ((0, [v["vc_document"] for v in issued], svc.verify_stored_vc_batch),
                               (1, [w["vc_document"] for w in wfs], svc.verify_stored_workflow_vc_batch)):
        mixed = _mix(docs, rng, foreign)
        raws = [m for m, _ in mixed]
        status, fields = svc._named_keyset().verify_stored(kind, raws)
        for (raw, want), st, f in zip(mixed, status, fields):
            exp = _expected(svc, kind, raw)
            if want is not None:
                assert st == want, (st, want, raw[:120])
            if st == HOST:
                continue
            assert st == exp, (st, exp, raw[:160])
            assert raw[f[0]:f[0] + f[1]].decode() == re.search(r'"issuer":"([^"]*)"', raw.decode()).group(1)
        assert sum(st == VALID for st in status) >= len(raws) // 2
        # the service: same verdicts and messages as the host path on every document
        res = verify(raws)
        for (raw, _), r in zip(mixed, res):
            exp = _expected(svc, kind, raw)
            assert r["valid"] == (exp == VALID), (r, exp)
            want_msg = {VALID: ("", "VC verified successfully"), INVALID: ("", "Invalid signature")}.get(exp)
            if want_msg:
                assert (r["error"], r["message"]) == want_msg
            elif exp == UNRESOLVED:
                assert r["error"] == "failed to resolve issuer DID: DID not found: %s" % foreign
            elif exp == BAD:
                assert r["error"].startswith("failed to verify signature: failed to decode signature: illegal base64 data at input byte ")
        # the same documents through the existing host path of the mirror (parse, re-marshal, keyed verify)
        if kind == 0:
            plain = [v for v in issued[:200]]
            assert [r["valid"] for r in verify([v["vc_document"] for v in plain])] == svc.verify_vc_batch(plain)
        else:
            assert [r["valid"] for r in verify(docs)] == svc.verify_workflow_vc_batch(wfs)
    assert _abi.VC_HOST == HOST


def test_host_and_device_calls_agree(ctx):
    import torch
    from agentfield_b200 import canonical as CA
    from agentfield_b200.identity import KeySet
    K, n = 16, 5000
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0xAFD7)
    from agentfield_b200 import ExpandedKeys
    cache = ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (4000 + a) for a in range(K)])
    d_exp = torch.from_numpy(cache._expanded).to(dev)
    d_ki = (torch.arange(n, device=dev) % K).to(torch.int32)
    d_docs, d_doff, d_msgs, d_moff, _ = CA.synthetic_stored_vcs_dev(ctx, d_exp, dids, d_ki, n, seed=3)
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    d_f = torch.empty((n, 4), dtype=torch.int32, device=dev)
    ks.verify_stored_dev(0, d_docs, d_doff, n, d_st, d_f)
    torch.cuda.synchronize()
    assert bool((d_st == VALID).all())
    buf, off = d_docs.cpu().numpy(), d_doff.cpu().numpy().view(np.uint64)
    st, fl = ks.verify_stored_packed(0, buf, off)
    assert (st == d_st.cpu().numpy()).all() and (fl == d_f.cpu().numpy().view(np.uint32)).all()
    docs = [buf[off[i]:off[i + 1]].tobytes() for i in range(n)]
    damaged = [d.replace(b'"proofValue":"', b'"proofValue":"A', 1) if i % 7 == 0 else d for i, d in enumerate(docs)]
    st2, _ = ks.verify_stored(0, damaged)
    assert ((st2 == INVALID) == (np.arange(n) % 7 == 0)).all()
    ks.close()


def test_chunk_boundaries_in_a_fresh_process():
    """The host-buffer call with chunks of 97 documents (AFC_CHUNK_ITEMS is read once per process)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, AFC_CHUNK_ITEMS="97", AFC_MIN_CHUNK_ITEMS="97")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(root, "tests", "test_vcdoc_gpu.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "test_host_and_device_calls_agree or test_stored_verdicts_equal_host_path_and_oracle"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "2 passed" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


def test_arguments_and_key_set_errors(ctx):
    from agentfield_b200 import _abi
    from agentfield_b200.identity import KeySet
    lib, h = _abi.load(), ctx.handle
    rng = np.random.default_rng(0xAFD8)
    pks = [CO.pubkey(rng.integers(0, 256, 32, dtype=np.uint8).tobytes()) for _ in range(3)]
    with pytest.raises(_abi.AfcError) as e:
        KeySet(pks, ctx, dids=["did:a", "did:b", "did:a"])
    assert e.value.rc == _abi.AFC_EINVAL
    plain = KeySet(pks, ctx)
    named = KeySet(pks, ctx, dids=["did:a", "did:b", "did:c"])
    doc = b"{}"
    off = np.array([0, 2], dtype=np.uint64)
    st = np.zeros(1, dtype=np.uint8)
    assert lib.afc_vc_verify_stored_batch(h, plain.handle, 0, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_ESTATE
    assert lib.afc_vc_verify_stored_batch(h, named.handle, 0, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == 0 and st[0] == HOST
    assert lib.afc_vc_verify_stored_batch(h, named.handle, 0, None, _abi.ptr(np.zeros(1, dtype=np.uint64)), 0, None, None) == 0     # empty batch
    assert lib.afc_vc_verify_stored_batch(h, named.handle, 2, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert lib.afc_vc_verify_stored_batch(h, named.handle, 0, doc, None, 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert lib.afc_vc_verify_stored_batch(h, named.handle, 0, None, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert lib.afc_vc_verify_stored_batch(h, None, 0, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert lib.afc_vc_verify_stored_batch(None, named.handle, 0, doc, _abi.ptr(off), 1, _abi.ptr(st), None) == _abi.AFC_EINVAL
    assert lib.afc_vc_verify_stored_batch_dev(h, named.handle, 0, None, None, 0, None, None, None) == _abi.AFC_EINVAL
    assert lib.afc_keyset_new_named(h, None, None, None, 0, C.byref(C.c_void_p())) == _abi.AFC_EINVAL
    plain.close(); named.close()


def test_one_million_documents(ctx):
    """1 M execution VCs from 1024 issuers built on the device, 1 % with a corrupted signature: the statuses are exactly the
    corruption pattern, and a sample equals the oracle's verification of the signing bytes the reference would build."""
    import torch
    from agentfield_b200 import canonical as CA
    from agentfield_b200.identity import KeySet
    n, K = 1 << 20, 1024
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0xAFD9)
    from agentfield_b200 import ExpandedKeys
    cache = ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (5000 + a) for a in range(K)])
    d_exp = torch.from_numpy(cache._expanded).to(dev)
    d_ki = (torch.arange(n, device=dev) % K).to(torch.int32)
    d_docs, d_doff, d_msgs, d_moff, d_sigs = CA.synthetic_stored_vcs_dev(ctx, d_exp, dids, d_ki, n, seed=11)
    bad = torch.arange(n, device=dev) % 100 == 37
    pv_at = d_doff[:-1] + (d_doff[1:] - d_doff[:-1]) - 3 - 40             # a character inside the proofValue (it ends 3 bytes early)
    d_docs[pv_at[bad]] = torch.where(d_docs[pv_at[bad]] == 0x41, 0x42, 0x41).to(torch.uint8)
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    ks.verify_stored_dev(0, d_docs, d_doff, n, d_st)
    torch.cuda.synchronize()
    assert torch.equal(d_st, torch.where(bad, INVALID, VALID).to(torch.uint8))
    m = 2000
    idx = np.unique(np.concatenate([np.arange(0, n, n // m), np.arange(37, n, 100)[:200]]))
    buf, off = d_docs.cpu().numpy(), d_doff.cpu().numpy()
    for i in idx[:400]:
        raw = buf[off[i]:off[i + 1]].tobytes()
        from agentfield_b200.services import go_unmarshal_vc
        from agentfield_b200 import go_json as GJ
        d = go_unmarshal_vc(raw, 0)
        msg = GJ.vc_document(d)
        sig = base64.urlsafe_b64decode(d["proof"]["proofValue"] + "==")
        ok = CO.ed25519_verify_batch(np.frombuffer(cache.public_key(d["issuer"]), dtype=np.uint8).reshape(1, 32),
                                     np.frombuffer(sig, dtype=np.uint8).reshape(1, 64), np.frombuffer(msg, dtype=np.uint8),
                                     np.array([0, len(msg)], dtype=np.uint64))[0]
        assert int(d_st[int(i)]) == (VALID if ok else INVALID), i
    ks.close()
