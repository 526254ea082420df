"""Stored credentials audited against their records on the GPU (afc_vc_audit_stored_batch, VCService.audit_stored_execution_vcs and
audit_workflow_chains): every result equals the host mirror (verify_execution_vc_comprehensive, verify_workflow_vc_comprehensive)
record for record, host-buffer and device calls agree (also across forced chunk boundaries), the argument errors, and a
1 M-record run whose masks are exactly the planted damage."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

VALID, INVALID, HOST, UNRESOLVED, BAD = 1, 0, 2, 3, 4
FOREIGN = "did:key:z" + "Q" * 46


def _service(ctx, n_issuers=32, seed=0xA0E1):
    from agentfield_b200 import ExpandedKeys
    from agentfield_b200.services import VCService
    rng = np.random.default_rng(seed)
    cache = ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (7000 + a) for a in range(n_issuers)])
    return cache, dids, VCService(cache, ctx)


def _record(r, v):
    return {"vc_id": r["vc_id"], "execution_id": r["execution_id"], "workflow_id": r["workflow_id"], "session_id": r["session_id"],
            "issuer_did": r["caller_did"], "target_did": r.get("target_did", ""), "caller_did": r["caller_did"], "vc_document": v["vc_document"],
            "signature": v["signature"], "input_hash": v["input_hash"], "output_hash": v["output_hash"], "status": r["status"]}


COLUMN_DAMAGE = {"issuer_did": "did:key:zOther", "execution_id": "exec-other", "workflow_id": "wf-other", "session_id": "", "caller_did": "did:key:z\xff",
                 "target_did": "t<&>", "status": "pending", "input_hash": "x", "output_hash": " ", "signature": "AAAA"}


def _damage(rec, i):
    """One kind of damage per record (i % 16): what the audit has to find, or nothing."""
    from agentfield_b200 import _abi
    rec = dict(rec)
    s = rec["vc_document"].decode("utf-8") if isinstance(rec["vc_document"], bytes) else rec["vc_document"]
    pv = re.search(r'"proofValue":"([^"]*)"', s).group(1)
    k = i % 16
    if k == 1:                                    # corrupted signature (the record keeps the original)
        j = 5 + i % 70
        s = s.replace(pv, pv[:j] + ("A" if pv[j] != "A" else "B") + pv[j + 1:])
    elif k == 2:                                  # value changed after signing, still canonical
        s = s.replace('"issuanceDate":"2', '"issuanceDate":"3', 1)
    elif k == 3:                                  # not the form json.Marshal writes: left to the host
        s = s.replace('"id":', '"id" :', 1)
    elif k == 4:                                  # unknown issuer
        s = re.sub(r'"issuer":"[^"]*"', '"issuer":"%s"' % FOREIGN, s, count=1)
    elif k == 5:                                  # undecodable proofValue
        s = s.replace(pv, pv[:7] + "+" + pv[8:])
    elif k == 6:                                  # one column of the record changed
        col = _abi.AUDIT_COLUMNS[(i // 16) % 10]
        rec[col] = COLUMN_DAMAGE[col]
    elif k == 7:                                  # statuses the device leaves to the host
        rec["status"] = ("\x1csucceeded", "o\u212a", "succeeded\x85", "ſucceeded")[(i // 16) % 4]      # U+212A: Kelvin sign
    elif k == 8:                                  # a timestamp the device leaves to the host (Arabic-Indic digits)
        s = re.sub(r'"issuanceDate":"\d', '"issuanceDate":"٢', s, count=1)
    elif k == 9:                                  # decodes, but not to 64 bytes
        s = s.replace(pv, pv[:40])
    elif k == 10:                                 # not JSON at all
        s = "{not json"
    elif k == 11:                                 # invalid timestamp, still canonical
        s = re.sub(r'"issuanceDate":"[^"]*"', '"issuanceDate":"2026-02-30T00:00:00Z"', s, count=1)
    elif k == 12:                                 # not W3C, not AgentField, missing id
        s = s.replace('"https://www.w3.org/2018/credentials/v1",', "", 1).replace('"AgentFieldExecutionCredential"', '"X"', 1)
        s = re.sub(r'"id":"[^"]*"', '"id":""', s, count=1)
    elif k == 13:                                 # status in another spelling, decided on the device
        same = (" Completed ", "OK", "success", "Succeeded\t") if rec["status"] == "succeeded" else (" Error ", "FAILURE", "errored", "Failed\n")
        rec["status"] = same[(i // 16) % 4]
    rec["vc_document"] = s if i % 2 else s.encode("utf-8")
    return rec


def _issued_records(ctx, svc, dids, n, rng):
    from test_host_logic import _vc_requests
    reqs = _vc_requests(n, dids, rng, pad_to=0)
    issued = svc.generate_execution_vc_batch(reqs)
    return [_record(r, v) for r, v in zip(reqs, issued)]


def test_audit_equals_mirror_record_for_record(ctx):
    from agentfield_b200 import _abi
    cache, dids, svc = _service(ctx)
    rng = np.random.default_rng(0xA0E2)
    recs = [_damage(r, i) for i, r in enumerate(_issued_records(ctx, svc, dids, 640, rng))]
    got = svc.audit_stored_execution_vcs(recs, "2026-10-01T00:00:00Z")
    want = [svc.verify_execution_vc_comprehensive(r, "2026-10-01T00:00:00Z") for r in recs]
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, i % 16, g, w)
    # the device decided most of them, and each path was taken
    docs = [r["vc_document"].encode() if isinstance(r["vc_document"], str) else r["vc_document"] for r in recs]
    st, iss = svc._named_keyset().audit_stored(0, docs, [[r[c] for c in _abi.AUDIT_COLUMNS] for r in recs])
    k = np.arange(len(recs)) % 16
    assert ((st == VALID) & (iss == 0)).sum() >= len(recs) // 4
    assert (st[k == 3] == HOST).all() and (st[k == 10] == HOST).all() and (st[k == 4] == UNRESOLVED).all() and (st[k == 5] == BAD).all()
    assert (iss[k == 7] & _abi.AUDIT_STATUS_UNDECIDED).all() and (iss[k == 8] & _abi.AUDIT_TIMESTAMP_UNDECIDED).all()
    assert (iss[k == 1] == 1 << 9).all() and (iss[k == 11] == _abi.AUDIT_INVALID_TIMESTAMP).all() and (iss[k == 13] == 0).all()
    for i in np.nonzero(k == 6)[0]:
        assert iss[i] == 1 << ((i // 16) % 10), (i, iss[i])
    assert all(g["valid"] for g, kk in zip(got, k) if kk in (0, 13)) and not any(g["valid"] for g, kk in zip(got, k) if kk in (1, 2, 4, 5, 6, 10))


def test_audit_workflow_chains_equal_mirror(ctx):
    cache, dids, svc = _service(ctx, seed=0xA0E3)
    rng = np.random.default_rng(0xA0E4)
    recs = _issued_records(ctx, svc, dids, 700, rng)
    chains, at = [], 0
    for c in range(200):
        m = c % 7
        comps = [_damage(r, at + j) if c % 3 == 0 else r for j, r in enumerate(recs[at:at + m])]
        at += m
        chains.append({"component_vcs": comps, "workflow_vc": None, "verification_timestamp": "t%d" % c})
    wfs = svc.generate_workflow_vc_batch([{"workflow_id": "wf-%d" % c, "root_did": dids[c % len(dids)], "vc_id": "v%d" % c, "workflow_vc_id": "w%d" % c,
                                           "issuance_date": "2026-09-22T00:00:00Z", "snapshot_time": "2026-09-22T00:00:00Z", "proof_created": "2026-09-22T00:00:01Z",
                                           "execution_vcs": [dict(e, created_at="2026-09-21T10:00:00Z") for e in ch["component_vcs"]
                                                             if isinstance(e["vc_document"], bytes) and e["vc_document"].startswith(b'{"@context"')]}
                                          for c, ch in enumerate(chains)])
    for c, (ch, wf) in enumerate(zip(chains, wfs)):
        if c % 5 == 4:
            continue                                   # no workflow VC
        doc = wf["vc_document"]
        if c % 5 == 1:
            doc = doc.replace(b'"snapshotTime":"2026-09-22', b'"snapshotTime":"2026-09-23', 1)          # tampered
        elif c % 5 == 2:
            doc = doc.replace(b'"AgentFieldWorkflowCredential"', b'"AgentFieldExecutionCredential"', 1)   # wrong type
        elif c % 10 == 3:
            doc = b" " + doc                                                                            # left to the host
        elif c % 10 == 8:
            doc = doc[:-3]                                                                              # does not parse
        ch["workflow_vc"] = dict(wf, vc_document=doc)
    got = svc.audit_workflow_chains(chains)
    for c, ch in enumerate(chains):
        w = svc.verify_workflow_vc_comprehensive(ch)
        assert got[c] == w, (c, got[c], w)
    assert sum(g["valid"] for g in got) > 40 and sum(not g["valid"] for g in got) > 40


def test_host_and_device_calls_agree(ctx):
    import torch
    from agentfield_b200 import ExpandedKeys, _abi, canonical as CA
    from agentfield_b200.identity import KeySet
    K, n = 16, 5000
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0xA0E5)
    cache = ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (8000 + a) for a in range(K)])
    d_exp = torch.from_numpy(cache._expanded).to(dev)
    d_ki = (torch.arange(n, device=dev) % K).to(torch.int32)
    d_docs, d_doff, _, _, _, d_cols, d_coff = CA.synthetic_stored_vcs_dev(ctx, d_exp, dids, d_ki, n, seed=5, audit_columns=True)
    d_cols[d_coff[10 * torch.arange(0, n, 11, device=dev) + 3]] ^= 1          # session_id of every 11th record
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    d_iss = torch.empty(n, dtype=torch.int32, device=dev)
    ks.audit_stored_dev(0, d_docs, d_doff, d_cols, d_coff, n, d_st, d_iss)
    torch.cuda.synchronize()
    want = np.where(np.arange(n) % 11 == 0, 1 << 3, 0)
    assert bool((d_st == VALID).all()) and (d_iss.cpu().numpy().view(np.uint32) == want).all()
    buf, off = d_docs.cpu().numpy(), d_doff.cpu().numpy().view(np.uint64)
    cbuf, coff = d_cols.cpu().numpy(), d_coff.cpu().numpy().view(np.uint64)
    st, iss = ks.audit_stored_packed(0, buf, off, cbuf, coff)
    assert (st == d_st.cpu().numpy()).all() and (iss == d_iss.cpu().numpy().view(np.uint32)).all()
    # the stored-verify call on the same documents gives the same statuses
    st_v, _ = ks.verify_stored_packed(0, buf, off)
    assert (st_v == st).all()
    # workflow documents: no columns
    wst, wiss = ks.audit_stored_packed(1, buf, off)
    assert (wst == HOST).all() and (wiss == 0).all()
    ks.close()
    assert _abi.AUDIT_COLUMNS[3] == "session_id"


def test_chunk_boundaries_in_a_fresh_process():
    """The host-buffer calls with chunks of 97 records (AFC_CHUNK_ITEMS is read once per process)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, AFC_CHUNK_ITEMS="97", AFC_MIN_CHUNK_ITEMS="97")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(root, "tests", "test_audit_gpu.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "test_host_and_device_calls_agree or test_audit_equals_mirror_record_for_record"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "2 passed" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


def test_argument_errors(ctx):
    from agentfield_b200 import _abi
    from agentfield_b200.identity import KeySet
    from oracle import c_oracle as CO
    lib, h = _abi.load(), ctx.handle
    rng = np.random.default_rng(0xA0E6)
    pks = [CO.pubkey(rng.integers(0, 256, 32, dtype=np.uint8).tobytes()) for _ in range(2)]
    plain = KeySet(pks, ctx)
    named = KeySet(pks, ctx, dids=["did:a", "did:b"])
    doc = b"{}"
    off = np.array([0, 2], dtype=np.uint64)
    cols = b"abcdefghij"
    coff = np.arange(11, dtype=np.uint64)
    st, iss = np.zeros(1, dtype=np.uint8), np.zeros(1, dtype=np.uint32)
    P = _abi.ptr
    call = lambda ks, kind, d, o, c, co, n, s, i: lib.afc_vc_audit_stored_batch(h, ks, kind, d, P(o), c, P(co), n, P(s), P(i))
    assert call(named.handle, 0, doc, off, cols, coff, 1, st, iss) == 0 and st[0] == HOST and iss[0] == 0
    assert call(plain.handle, 0, doc, off, cols, coff, 1, st, iss) == _abi.AFC_ESTATE
    assert call(named.handle, 0, doc, off, None, None, 1, st, iss) == _abi.AFC_EINVAL        # execution batch without columns
    assert call(named.handle, 0, doc, off, cols, None, 1, st, iss) == _abi.AFC_EINVAL
    assert call(named.handle, 1, doc, off, cols, coff, 1, st, iss) == _abi.AFC_EINVAL        # workflow batch with columns
    assert call(named.handle, 1, doc, off, None, None, 1, st, iss) == 0 and st[0] == HOST
    assert call(named.handle, 2, doc, off, None, None, 1, st, iss) == _abi.AFC_EINVAL        # bad kind
    assert call(named.handle, 0, None, off, cols, coff, 1, st, iss) == _abi.AFC_EINVAL
    assert call(named.handle, 0, doc, None, cols, coff, 1, st, iss) == _abi.AFC_EINVAL
    assert call(named.handle, 0, doc, off, cols, coff, 1, None, iss) == _abi.AFC_EINVAL
    assert call(named.handle, 0, doc, off, cols, coff, 1, st, None) == _abi.AFC_EINVAL
    assert call(None, 0, doc, off, cols, coff, 1, st, iss) == _abi.AFC_EINVAL
    assert lib.afc_vc_audit_stored_batch(None, named.handle, 0, doc, P(off), cols, P(coff), 1, P(st), P(iss)) == _abi.AFC_EINVAL
    bad = coff.copy(); bad[5], bad[6] = 6, 5                                                  # column offsets running backwards
    assert call(named.handle, 0, doc, off, cols, bad, 1, st, iss) == _abi.AFC_EINVAL
    assert call(named.handle, 0, None, np.zeros(1, dtype=np.uint64), None, np.zeros(1, dtype=np.uint64), 0, None, None) == 0   # empty batch
    assert lib.afc_vc_audit_stored_batch_dev(h, named.handle, 0, None, None, None, None, 0, None, None, None) == _abi.AFC_EINVAL
    assert lib.afc_vc_audit_stored_batch_dev(h, plain.handle, 1, None, P(off), None, None, 0, None, None, None) == _abi.AFC_ESTATE
    plain.close(); named.close()


def test_one_million_records(ctx):
    """2^20 records from 1024 issuers built on the device; 1 % with a corrupted signature, 1 % with one column of the record changed
    (over all ten columns): every status and every mask is exactly the planted damage."""
    import torch
    from agentfield_b200 import ExpandedKeys, canonical as CA
    from agentfield_b200.identity import KeySet
    n, K = 1 << 20, 1024
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(0xA0E7)
    cache = ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (9000 + a) for a in range(K)])
    d_exp = torch.from_numpy(cache._expanded).to(dev)
    d_ki = (torch.arange(n, device=dev) % K).to(torch.int32)
    d_docs, d_doff, _, _, _, d_cols, d_coff = CA.synthetic_stored_vcs_dev(ctx, d_exp, dids, d_ki, n, seed=13, audit_columns=True)
    want_st, want_iss = plant_damage(d_docs, d_doff, d_cols, d_coff, n)
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    d_iss = torch.empty(n, dtype=torch.int32, device=dev)
    ks.audit_stored_dev(0, d_docs, d_doff, d_cols, d_coff, n, d_st, d_iss)
    torch.cuda.synchronize()
    assert torch.equal(d_st, want_st) and torch.equal(d_iss, want_iss)
    ks.close()


def plant_damage(d_docs, d_doff, d_cols, d_coff, n):
    """Corrupts a proofValue character of 1 % of the documents and one byte of one column of another 1 % of the records (column
    (i // 100) % 10); returns the expected statuses and masks (int32 view of the uint32 masks)."""
    import torch
    dev = d_docs.device
    i = torch.arange(n, device=dev)
    bad_sig = i % 100 == 37
    pv_at = d_doff[1:] - 3 - 40                                      # inside proofValue (the document ends with "}})
    d_docs[pv_at[bad_sig]] = torch.where(d_docs[pv_at[bad_sig]] == 0x41, 0x42, 0x41).to(torch.uint8)
    bad_col = i % 100 == 53
    k = (i // 100) % 10
    at = d_coff[10 * i[bad_col] + k[bad_col]]
    d_cols[at] ^= 1
    want_st = torch.where(bad_sig, INVALID, VALID).to(torch.uint8)
    want_iss = torch.zeros(n, dtype=torch.int32, device=dev)
    want_iss[bad_sig] = 1 << 9                                       # the record keeps the signature it was issued with
    want_iss[bad_col] = (1 << k[bad_col]).to(torch.int32)
    return want_st, want_iss
