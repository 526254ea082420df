#!/usr/bin/env python
"""Stored execution-VC documents verified from their bytes (afc_vc_verify_stored_batch[_dev]) against the keyed-verify floor.
Prints one JSON line: documents/s of the device-pointer call with its per-kernel split, of the keyed verify alone over the same
signing bytes already rendered, and of the host-buffer call; host_fallback and all_expected; the card and its power limit, read
in the same run.  The audit_stored block does the same for the audit of stored execution VCs against their records
(afc_vc_audit_stored_batch[_dev]), next to the stored-verify device call on the same documents.  The verify_json block measures
documents in three client spellings (afc_vc_verify_json_batch_dev) next to the stored-verify call on the canonical form.  The
issue_execution block measures execution credentials issued in one call (afc_vc_issue_execution_batch[_dev]).  The webhook block
measures webhook deliveries built and signed in one call (afc_webhook_sign_batch[_dev]) next to HMAC alone over the same bodies.
The issue_workflow block measures workflow credentials issued in one call (afc_vc_issue_workflow_batch[_dev]) next to the host-built path.
The reregister block measures known agents re-registered in one call (afc_did_reregister_batch[_dev]) in a restart storm.
Needs a CUDA device; writes nothing.
usage: python tools/bench_stored_vc.py [--reps R] [--only BLOCK]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def stored_vc_block(ctx, dev, timed):
    """Stored execution-VC documents verified from their bytes (afc_vc_verify_stored_batch): 2^20 documents of ~1.3 KB from 1024
    issuers, built on the device (template fill + expanded-key signing), 1 % with a corrupted signature.  Against the floor: the
    keyed verify alone over the same signing bytes, already rendered.  host_fallback counts documents the device left to the host
    (0 expected: these are exactly what json.Marshal writes)."""
    import torch
    import agentfield_b200 as afb
    from agentfield_b200 import canonical as CA
    from agentfield_b200.identity import KeySet
    n, K = 1 << 20, 1024
    rng = np.random.default_rng(0xAF07)
    cache = afb.ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (6000 + a) for a in range(K)])
    d_exp = torch.from_numpy(cache._expanded).to(dev)
    d_ki = (torch.arange(n, device=dev) % K).to(torch.int32)
    d_docs, d_doff, d_msgs, d_moff, d_sigs = CA.synthetic_stored_vcs_dev(ctx, d_exp, dids, d_ki, n, seed=0xAF07)
    bad = torch.arange(n, device=dev) % 100 == 37
    pv_at = d_doff[1:] - 3 - 40                                      # inside proofValue (the document ends with "}})
    d_docs[pv_at[bad]] = torch.where(d_docs[pv_at[bad]] == 0x41, 0x42, 0x41).to(torch.uint8)
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    d_f = torch.empty((n, 4), dtype=torch.int32, device=dev)
    run = lambda: ks.verify_stored_dev(0, d_docs, d_doff, n, d_st, d_f)
    ms_dev = timed(run)
    expect = torch.where(bad, 0, 1).to(torch.uint8)
    all_expected = bool(torch.equal(d_st, expect))
    host_fallback = int((d_st == 2).sum())
    ctx.profile_begin()
    timed(run, reps=3)
    kms = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
    d_ok = torch.empty(n, dtype=torch.uint8, device=dev)
    ms_floor = timed(lambda: ks.verify_dev(d_ki, d_sigs, d_msgs, d_moff, n, d_ok))
    buf, off = d_docs.cpu().numpy(), d_doff.cpu().numpy().view(np.uint64)
    st_host = np.empty(n, dtype=np.uint8)
    fl_host = np.empty((n, 4), dtype=np.uint32)
    lib, P = afb._abi.load(), afb._abi.ptr

    def host_call():
        afb._abi.check(lib.afc_vc_verify_stored_batch(ctx.handle, ks.handle, 0, P(buf), P(off), n, P(st_host), P(fl_host)))
    host_call()
    t0 = time.perf_counter()
    for _ in range(3):
        host_call()
    ms_host = (time.perf_counter() - t0) / 3 * 1e3
    all_expected = all_expected and bool((st_host == expect.cpu().numpy()).all())
    ks.close()
    gpu = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return {"docs": n, "issuers": K, "bytes": int(off[-1]), "avg_doc_bytes": int(off[-1]) / n, "gpu": gpu,
            "dev_call": {"docs_per_s": n / (ms_dev * 1e-3), "ms": ms_dev, "kernels_ms": kms},
            "keyed_verify_floor": {"docs_per_s": n / (ms_floor * 1e-3), "ms": ms_floor,
                                   "note": "afc_ed25519_verify_keyed_batch_dev over the same signing bytes, pre-rendered"},
            "host_call": {"docs_per_s": n / (ms_host * 1e-3), "ms": ms_host, "note": "documents in pageable host memory, statuses and fields back"},
            "host_fallback": host_fallback, "all_expected": all_expected}


def audit_stored_block(ctx, dev, timed):
    """Stored execution VCs audited against their records (afc_vc_audit_stored_batch): 2^20 records from 1024 issuers built on the
    device, 1 % with a corrupted signature, 1 % with one column of the record changed (over all ten columns).  Beside it, the
    stored-verify device call on the same documents.  all_expected: every status and every mask is exactly the planted damage;
    host_fallback / undecided count documents and masks the host would have to finish (0 expected)."""
    import torch
    import agentfield_b200 as afb
    from agentfield_b200 import canonical as CA
    from agentfield_b200.identity import KeySet
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_audit_gpu import plant_damage
    n, K = 1 << 20, 1024
    rng = np.random.default_rng(0xAF08)
    cache = afb.ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (6000 + a) for a in range(K)])
    d_exp = torch.from_numpy(cache._expanded).to(dev)
    d_ki = (torch.arange(n, device=dev) % K).to(torch.int32)
    d_docs, d_doff, _, _, _, d_cols, d_coff = CA.synthetic_stored_vcs_dev(ctx, d_exp, dids, d_ki, n, seed=0xAF08, audit_columns=True)
    want_st, want_iss = plant_damage(d_docs, d_doff, d_cols, d_coff, n)
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    d_iss = torch.empty(n, dtype=torch.int32, device=dev)
    run = lambda: ks.audit_stored_dev(0, d_docs, d_doff, d_cols, d_coff, n, d_st, d_iss)
    ms_dev = timed(run)
    all_expected = bool(torch.equal(d_st, want_st)) and bool(torch.equal(d_iss, want_iss))
    host_fallback = int((d_st == 2).sum())
    undecided = int(((d_iss & ((1 << 18) | (1 << 19))) != 0).sum())
    ctx.profile_begin()
    timed(run, reps=3)
    kms = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
    d_st2 = torch.empty(n, dtype=torch.uint8, device=dev)
    verify = lambda: ks.verify_stored_dev(0, d_docs, d_doff, n, d_st2)
    ms_verify = timed(verify)
    ctx.profile_begin()
    timed(verify, reps=3)
    vkms = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
    buf, off = d_docs.cpu().numpy(), d_doff.cpu().numpy().view(np.uint64)
    cbuf, coff = d_cols.cpu().numpy(), d_coff.cpu().numpy().view(np.uint64)
    st_host = np.empty(n, dtype=np.uint8)
    iss_host = np.empty(n, dtype=np.uint32)
    lib, P = afb._abi.load(), afb._abi.ptr

    def host_call():
        afb._abi.check(lib.afc_vc_audit_stored_batch(ctx.handle, ks.handle, 0, P(buf), P(off), P(cbuf), P(coff), n, P(st_host), P(iss_host)))
    host_call()
    t0 = time.perf_counter()
    for _ in range(3):
        host_call()
    ms_host = (time.perf_counter() - t0) / 3 * 1e3
    all_expected = all_expected and bool((st_host == want_st.cpu().numpy()).all()) and bool((iss_host == want_iss.cpu().numpy().view(np.uint32)).all())
    ks.close()
    gpu = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return {"records": n, "issuers": K, "doc_bytes": int(off[-1]), "column_bytes": int(coff[-1]), "gpu": gpu,
            "dev_call": {"docs_per_s": n / (ms_dev * 1e-3), "ms": ms_dev, "kernels_ms": kms},
            "stored_verify_dev_call": {"docs_per_s": n / (ms_verify * 1e-3), "ms": ms_verify, "kernels_ms": vkms,
                                       "note": "afc_vc_verify_stored_batch_dev on the same documents"},
            "host_call": {"docs_per_s": n / (ms_host * 1e-3), "ms": ms_host, "note": "documents and columns in pageable host memory, statuses and masks back"},
            "host_fallback": host_fallback, "undecided": undecided, "all_expected": all_expected}


def verify_json_block(ctx, dev, timed):
    """Documents in any JSON spelling re-marshalled on the device (afc_vc_verify_json_batch): 2^20 execution VCs from 1024 issuers,
    1 % with a corrupted signature, in three spellings: the canonical bytes, json.dumps(doc, indent=2, ensure_ascii=False) (the shape
    of JSON.stringify(doc, null, 2)) and json.dumps(doc) (what requests sends).  2^16 distinct documents are built on the device,
    re-spelled on the host with every number token kept, tiled to 2^20, then corrupted.  Beside them, the stored-verify call on the
    canonical form.  host_fallback must be 0 and all_expected true for every spelling."""
    import torch
    from agentfield_b200.respell import respelled_stored_vcs_dev
    n, K = 1 << 20, 1024
    out = {"docs": n, "issuers": K}
    for name, how in (("canonical", None), ("indent2_no_ascii", "js_pretty"), ("dumps", "dumps")):
        d_docs, d_off, ks, want = respelled_stored_vcs_dev(ctx, dev, n, K, 0xAF09, how)
        d_st = torch.empty(n, dtype=torch.uint8, device=dev)
        run = lambda: ks.verify_json_dev(0, d_docs, d_off, n, d_st)
        ms = timed(run)
        r = {"bytes": int(d_off[-1]), "docs_per_s": n / (ms * 1e-3), "ms": ms, "host_fallback": int((d_st == 2).sum()),
             "all_expected": bool(torch.equal(d_st, want))}
        ctx.profile_begin()
        timed(run, reps=3)
        r["kernels_ms"] = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
        if how is None:
            d_st2 = torch.empty(n, dtype=torch.uint8, device=dev)
            stored = lambda: ks.verify_stored_dev(0, d_docs, d_off, n, d_st2)
            ms_s = timed(stored)
            ctx.profile_begin()
            timed(stored, reps=3)
            out["stored_dev_call"] = {"docs_per_s": n / (ms_s * 1e-3), "ms": ms_s, "all_expected": bool(torch.equal(d_st2, want)),
                                      "kernels_ms": {k: v["avg_ms"] for k, v in ctx.profile_end().items()},
                                      "note": "afc_vc_verify_stored_batch_dev on the canonical documents"}
        out[name] = r
        ks.close()
        del d_docs, d_off
    out["gpu"] = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    return out


def issue_execution_block(ctx, dev, timed):
    """Execution credentials issued on the device (afc_vc_issue_execution_batch): 2^20 requests from 1024 issuers (55-character DIDs,
    RFC 3339 times), input and output payloads of 64-2048 B (uniform, seeded; 10 % nil), 1 % with an error message that needs escaping
    (a third of those past 500 bytes), constant-time signing.  Next to it, the same device work done the way the service did it before:
    SHA-256 over the pre-encoded payload text, the template fill without proof, expanded-key signing, base64url, the fill with proof.
    Also the host-buffer call (2^18 requests, pinned buffers), the _dev call appending to a log, and a tail variant where 0.1 % of the
    payloads are 256 KiB.  Every hash and every signature is checked (hashlib; afc_vc_verify_stored_batch), and 2000 sampled documents
    byte for byte against the host mirror, before timing."""
    import base64
    import hashlib
    import torch
    import agentfield_b200 as afb
    from agentfield_b200 import canonical as CA, go_json, services
    from agentfield_b200.identity import KeySet
    n, K = 1 << 20, 1024
    rng = np.random.default_rng(0xAF1E)
    cache = afb.ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (8000 + a) for a in range(K)])
    d_exp = torch.from_numpy(cache._expanded).to(dev)
    t = lambda a: torch.from_numpy(a).to(dev)

    def upload(reqs):
        cols, coff, dur, pay, poff, nil = cache.pack_issue_requests(reqs)
        ki = cache.key_index([r["caller_did"] for r in reqs])
        return dict(d_key_index=t(ki.view(np.int32)), d_cols=t(cols), d_col_off=t(coff.view(np.int64)), d_duration=t(dur), d_payloads=t(pay),
                    d_payload_off=t(poff.view(np.int64)), d_payload_nil=t(nil), n=len(reqs), d_expanded=d_exp), (cols, coff, dur, pay, poff, nil, ki)
    reqs = CA.synthetic_issue_requests(dids, n, seed=0xAF1E)
    D, H = upload(reqs)
    pay_bytes = int(H[4][-1])
    d_docs, d_off, d_h, d_pv = cache.issue_dev(**D)
    torch.cuda.synchronize()
    # checks: every hash (hashlib), every document (verify), 2000 documents byte for byte (host mirror)
    h = d_h.cpu().numpy()
    hashes_ok = True
    for i, r in enumerate(reqs):
        for k, d in ((0, r["input"]), (1, r["output"])):
            m = services.marshal_data_or_null(None if d is None else bytes(d))
            hashes_ok &= h[i, 43 * k:43 * k + 43].tobytes() == base64.urlsafe_b64encode(hashlib.sha256(m).digest()).rstrip(b"=")
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    ks.verify_stored_dev(0, d_docs, d_off, n, d_st)
    verify_ok = bool((d_st == 1).all())
    ks.close()
    docs_host, off_host, pv = d_docs.cpu().numpy().tobytes(), d_off.cpu().numpy(), d_pv.cpu().numpy()
    sample = rng.choice(n, 2000, replace=False)
    svc = services.VCService(cache, canonical_on_device=False)
    mirror = svc.generate_execution_vc_batch([reqs[int(i)] for i in sample])
    sample_ok = all(m["vc_document"] == docs_host[int(off_host[i]):int(off_host[i + 1])] and m["signature"] == pv[i].tobytes().decode()
                    for m, i in zip(mirror, sample))
    all_expected = bool(hashes_ok and verify_ok and sample_ok)
    run = lambda: cache.issue_dev(**D)
    ms_dev = timed(run)
    ctx.profile_begin()
    timed(run, reps=3)
    kms = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
    total_bytes = int(off_host[-1])
    # the same device work the way the service did it before: hash pre-encoded text, fill, sign, base64url, fill again
    text = [services.marshal_data_or_null(None if r[k] is None else bytes(r[k])) for r in reqs for k in ("input", "output")]
    tbuf, toff = afb.crypto.pack(text)
    del text
    d_tbuf, d_toff = t(tbuf), t(toff.view(np.int64))
    d_dig = torch.empty((2 * n, 32), dtype=torch.uint8, device=dev)
    t0, t1 = CA.vc_document_template(False, ctx), CA.vc_document_template(True, ctx)
    ctxlist, typelist = go_json.string_list(["https://www.w3.org/2018/credentials/v1", "https://agentfield.example.com/contexts/execution/v1"]).encode(), \
        go_json.string_list(["VerifiableCredential", "AgentFieldExecutionCredential"]).encode()
    md = b'{"agentfield_version":"1.0.0","vc_version":"1.0"}'
    u = lambda s: s.encode("utf-8", "surrogatepass")
    v0, v1 = [], []
    for i, r in enumerate(reqs):
        ih, oh = h[i, :43].tobytes(), h[i, 43:].tobytes()
        em = go_json.truncate_error_message(r["error_message"])
        row = [ctxlist, typelist, b"urn:agentfield:vc:" + u(r["vc_id"]), u(r["caller_did"]), u(r["issuance_date"]), u(r["execution_id"]),
               u(r["workflow_id"]), u(r["session_id"]), u(r["caller_did"]), u(r["caller_type"]), u(r["agent_node_did"]), u(r["target_did"]),
               u(r["agent_node_did"]), u(r["function_name"]), ih, oh, u(r["timestamp"]), b"%d" % r["duration_ms"], u(r["status"]),
               (b',"errorMessage":' + go_json.any_string(em).encode("utf-8")) if em else b"", ih, oh, md]
        v0.append(row)
        v1.append(row + [b"Ed25519Signature2020", u(r["proof_created"]), u(r["caller_did"]) + b"#key-1", b"assertionMethod", pv[i].tobytes()])
    f0, o0 = t0.pack_values(v0)
    f1, o1 = t1.pack_values(v1)
    del v0, v1
    d_f0, d_o0, d_f1, d_o1 = t(f0), t(o0.view(np.int64)), t(f1), t(o1.view(np.int64))
    d_sigs = torch.empty((n, 64), dtype=torch.uint8, device=dev)
    d_pv2 = torch.empty((n, 86), dtype=torch.uint8, device=dev)
    ms_sha = timed(lambda: ctx.sha256_dev(d_tbuf, d_toff, 2 * n, d_dig))
    ms_fill0 = timed(lambda: t0.fill_dev(d_f0, d_o0, n))
    d_msgs, d_moff = t0.fill_dev(d_f0, d_o0, n)
    ms_sign = timed(lambda: ctx.sign_expanded_dev(d_exp, D["d_key_index"], d_msgs, d_moff, n, d_sigs))
    ms_b64 = timed(lambda: ctx.b64url_encode_dev(d_sigs, 64, n, d_pv2))
    ms_fill1 = timed(lambda: t1.fill_dev(d_f1, d_o1, n))
    d_docs1, _ = t1.fill_dev(d_f1, d_o1, n)
    pieces_same = bool(torch.equal(d_pv2, d_pv)) and bool(torch.equal(d_docs1, d_docs))
    del d_tbuf, d_toff, d_dig, d_f0, d_o0, d_f1, d_o1, d_msgs, d_moff, d_docs1, tbuf, f0, f1
    # the _dev call appending to a log
    aud = afb.Auditor(ctx)
    ms_log = timed(lambda: cache.issue_dev(**D, log=aud))
    aud.close()
    del d_docs, d_off, d_h, d_pv
    # the host-buffer call, pinned buffers, 2^18 requests
    nh = 1 << 18
    cols, coff, dur, pay, poff, nil, ki = H
    cut_c, cut_p = int(coff[nh * 14]), int(poff[2 * nh])

    def pin(a):
        p = torch.empty(a.shape, dtype=torch.from_numpy(a[:0]).dtype, pin_memory=True).numpy()
        p[...] = a
        return p
    hin = [pin(cols[:cut_c]), pin(coff[:nh * 14 + 1]), pin(dur[:nh]), pin(pay[:cut_p]), pin(poff[:2 * nh + 1]), pin(nil[:2 * nh])]
    lib, P = afb._abi.load(), afb._abi.ptr
    cap = lib.afc_vc_issue_bound(P(hin[1]), nh)
    hdocs = torch.empty(cap, dtype=torch.uint8, pin_memory=True).numpy()
    hoff = torch.empty(nh + 1, dtype=torch.int64, pin_memory=True).numpy()
    hh = torch.empty((nh, 86), dtype=torch.uint8, pin_memory=True).numpy()
    hpv = torch.empty((nh, 86), dtype=torch.uint8, pin_memory=True).numpy()
    hki = pin(ki[:nh])

    def host_call():
        afb._abi.check(lib.afc_vc_issue_execution_batch(ctx.handle, P(cache._expanded), K, P(hki), P(hin[0]), P(hin[1]), P(hin[2]), P(hin[3]),
                                                        P(hin[4]), P(hin[5]), afb._abi.ISSUE_HASH_DATA, nh, None, P(hdocs), cap, P(hoff), P(hh),
                                                        P(hpv)), ctx.handle)
    host_call()
    host_same = hoff[nh] == off_host[nh] and hdocs[:hoff[nh]].tobytes() == docs_host[:int(off_host[nh])] and (hpv == pv[:nh]).all() and \
        (hh == h[:nh]).all()
    t_0 = time.perf_counter()
    for _ in range(3):
        host_call()
    ms_host = (time.perf_counter() - t_0) / 3 * 1e3
    del hin, hdocs, hoff, hh, hpv, hki, H, D
    torch.cuda.empty_cache()
    # tail: 0.1 % of the payloads are 256 KiB
    treqs = CA.synthetic_issue_requests(dids, n, seed=0xAF1F, long_frac=0.001)
    TD, _ = upload(treqs)
    long_n = sum((r["input"] is not None and len(r["input"]) == 256 << 10) + (r["output"] is not None and len(r["output"]) == 256 << 10) for r in treqs)
    d_docs, d_off, d_h, d_pv = cache.issue_dev(**TD)
    torch.cuda.synchronize()
    th = d_h.cpu().numpy()
    tail_ok = True
    for i in range(0, n, 97):
        r = treqs[i]
        for k, d in ((0, r["input"]), (1, r["output"])):
            m = services.marshal_data_or_null(None if d is None else bytes(d))
            tail_ok &= th[i, 43 * k:43 * k + 43].tobytes() == base64.urlsafe_b64encode(hashlib.sha256(m).digest()).rstrip(b"=")
    del d_docs, d_off, d_h, d_pv
    ms_tail = timed(lambda: cache.issue_dev(**TD))
    ctx.profile_begin()
    timed(lambda: cache.issue_dev(**TD), reps=3)
    tkms = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
    gpu = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    old = ms_sha + ms_fill0 + ms_sign + ms_b64 + ms_fill1
    return {"requests": n, "issuers": K, "payload_bytes": pay_bytes, "doc_bytes": total_bytes, "gpu": gpu,
            "all_expected": all_expected, "hashes_ok": bool(hashes_ok), "verify_ok": verify_ok, "sample_ok": bool(sample_ok),
            "dev_call": {"vcs_per_s": n / (ms_dev * 1e-3), "ms": ms_dev, "kernels_ms": kms},
            "pieces": {"ms": old, "vcs_per_s": n / (old * 1e-3), "sha256_ms": ms_sha, "fill_ms": ms_fill0, "sign_ms": ms_sign, "b64url_ms": ms_b64,
                       "fill_proof_ms": ms_fill1, "same_bytes": pieces_same,
                       "note": "afc_sha256_batch_dev over pre-encoded text, two template fills, expanded-key signing, base64url; host work not counted"},
            "dev_call_with_log": {"vcs_per_s": n / (ms_log * 1e-3), "ms": ms_log},
            "host_call": {"requests": nh, "vcs_per_s": nh / (ms_host * 1e-3), "ms": ms_host, "same_as_dev": bool(host_same),
                          "note": "every buffer pinned"},
            "tail": {"long_payloads": int(long_n), "vcs_per_s": n / (ms_tail * 1e-3), "ms": ms_tail, "kernels_ms": tkms, "hashes_ok": bool(tail_ok)}}


def webhook_results(count, seed):
    """Agent results as the Python SDK stores them: json.dumps default spelling of nested objects of 100 B - 4 KB, keys in insertion
    (unsorted) order, 17-digit floats, non-ASCII text as \\u escapes in values."""
    import random
    rng = random.Random(seed)

    def val(depth):
        k = rng.random()
        if depth < 3 and k < 0.2:
            return {"k%02d_%s" % (rng.randrange(100), rng.choice(["score", "label", "items", "meta"])): val(depth + 1) for _ in range(rng.randrange(1, 6))}
        if depth < 3 and k < 0.3:
            return [val(depth + 1) for _ in range(rng.randrange(1, 5))]
        if k < 0.55:
            return rng.random() * 10.0 ** rng.randrange(-5, 8)
        if k < 0.65:
            return rng.randrange(-10 ** 9, 10 ** 9)
        if k < 0.9:
            return "".join(rng.choice("abcdefghij <>&é中😀\n") for _ in range(rng.randrange(4, 40)))
        return rng.choice([True, False, None])
    out = []
    while len(out) < count:
        target = int(100 * 40 ** rng.random())                  # 100 B - 4 KB, log-uniform
        d = {}
        while len(json.dumps(d)) < target:
            d["field_%d_%s" % (rng.randrange(1000), rng.choice(["answer", "score", "trace"]))] = val(0)
        out.append(json.dumps(d).encode())
    return out


def webhook_block(ctx, dev, timed):
    """afc_webhook_sign_batch_dev over 2^20 deliveries: results drawn from 4096 seeded texts, 10 % failed deliveries with error messages,
    10 % without a secret, 1 % planted AFC_WEBHOOK_HOST (a status with a non-ASCII space)."""
    import random
    import torch
    import agentfield_b200 as afb
    from agentfield_b200 import go_json, services
    n = 1 << 20
    texts = webhook_results(4096, 0xAF20)
    rng = random.Random(0xAF21)
    base = []
    for i in range(4096):
        failed = i % 10 == 3
        base.append(dict(execution_id="exec_%07d" % i, run_id="run_%05d" % (i // 7), status="failed" if failed else "succeeded", node_id="agent-%d" % (i % 97),
                         reasoner_id="reasoner_%d" % (i % 13), target_type="reasoner", timestamp="2026-09-21T06:%02d:%02dZ" % (i // 60 % 60, i % 60),
                         duration_ms=rng.randrange(0, 10 ** 6), result=texts[i], error_message="step %d failed: <timeout> & retry" % i if failed else None,
                         secret=None if i % 10 == 7 else "whsec_%032x" % rng.getrandbits(128)))
    recs = []
    planted = 0
    for i in range(n):
        r = base[i % 4096]
        if i % 100 == 51:
            r = dict(r, status="done\x85")
            planted += 1
        recs.append(r)
    packed = services.pack_webhook_deliveries(recs)
    cb, co, dur, fl, rb, ro, sb, so = packed
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    lib, P = afb._abi.load(), afb._abi.ptr
    cap = int(lib.afc_webhook_bound(P(co), P(ro), n))
    D = [t(cb), t(co.view(np.int64)), t(dur), t(fl), t(rb), t(ro.view(np.int64)), t(sb), t(so.view(np.int32))]
    d_bodies = torch.empty(cap, dtype=torch.uint8, device=dev)
    d_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    d_h = torch.empty((n, 71), dtype=torch.uint8, device=dev)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)

    def dev_call():
        ctx.webhook_sign_dev(*D, n, d_bodies, cap, d_off, d_h, d_st)
    dev_call()
    torch.cuda.synchronize()
    st = d_st.cpu().numpy()
    off = d_off.cpu().numpy().view(np.uint64)
    host_fallback = int((st == afb._abi.WEBHOOK_HOST).sum())
    bodies = d_bodies[:int(off[-1])].cpu().numpy()
    srng = random.Random(3)
    sample_ok = all(st[i] == afb._abi.WEBHOOK_HOST or bodies[int(off[i]):int(off[i + 1])].tobytes() == go_json.build_webhook_payload(recs[i])
                    for i in srng.sample(range(n), 2000))
    ms_dev = timed(dev_call)
    ctx.profile_begin()
    timed(dev_call, reps=3)
    kms = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
    # the floor: HMAC alone over the same bodies, built beforehand
    d_sec, d_soff = D[6], D[7]
    d_mac = torch.empty((n, 32), dtype=torch.uint8, device=dev)
    ms_hmac = timed(lambda: ctx.hmac_sha256_dev(d_sec, d_soff, d_bodies, d_off, n, d_mac))
    body_bytes = int(off[-1])
    del d_bodies, d_h, d_mac, D
    torch.cuda.empty_cache()
    # the host-buffer call from pinned memory
    nh = 1 << 18

    def pin(a):
        p_ = torch.empty(a.shape, dtype=torch.from_numpy(a[:0]).dtype, pin_memory=True).numpy()
        p_[...] = a
        return p_
    hp = services.pack_webhook_deliveries(recs[:nh])
    hin = [pin(a) for a in hp]
    hcap = int(lib.afc_webhook_bound(P(hin[1]), P(hin[5]), nh))
    hb = torch.empty(hcap, dtype=torch.uint8, pin_memory=True).numpy()
    hoff = torch.empty(nh + 1, dtype=torch.int64, pin_memory=True).numpy()
    hh = torch.empty((nh, 71), dtype=torch.uint8, pin_memory=True).numpy()
    hs = torch.empty(nh, dtype=torch.uint8, pin_memory=True).numpy()

    def host_call():
        afb._abi.check(lib.afc_webhook_sign_batch(ctx.handle, *[P(a) for a in hin], nh, P(hb), hcap, P(hoff), P(hh), P(hs)), ctx.handle)
    host_call()
    host_same = int(hoff[nh]) == int(off[nh]) and hb[:int(hoff[nh])].tobytes() == bodies[:int(off[nh])].tobytes()
    t_0 = time.perf_counter()
    for _ in range(3):
        host_call()
    ms_host = (time.perf_counter() - t_0) / 3 * 1e3
    gpu = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return {"deliveries": n, "result_bytes": int(ro[-1]), "body_bytes": body_bytes, "gpu": gpu, "planted_host": planted, "host_fallback": host_fallback,
            "sample_ok": bool(sample_ok), "dev_call": {"deliveries_per_s": n / (ms_dev * 1e-3), "ms": ms_dev, "kernels_ms": kms},
            "hmac_floor": {"deliveries_per_s": n / (ms_hmac * 1e-3), "ms": ms_hmac, "note": "afc_hmac_sha256_batch_dev over the bodies, built beforehand"},
            "host_call": {"deliveries": nh, "deliveries_per_s": nh / (ms_host * 1e-3), "ms": ms_host, "same_as_dev": bool(host_same),
                          "note": "every buffer pinned"}}


def issue_workflow_block(ctx, dev, timed):
    """Workflow credentials issued on the device (afc_vc_issue_workflow_batch): 2^16 workflows of 1-64 records each (~2^21 records) from
    1024 issuers, ids shaped like generateVCID's vc-<nanos>, a status mix of mostly succeeded with failed, running, cancelled, timeout,
    queued and pending records and aliases; then a skewed batch in which 1 % of the workflows hold 4096 records.  Next to them, the
    host-built path (generate_workflow_vc_batch: documents in Python, signatures in one GPU batch) on 2000 of the workflows, whose documents
    must equal the device's byte for byte, and the host-buffer call from unpinned numpy arrays.  Every device document is verified
    (afc_vc_verify_stored_batch) before timing."""
    import torch
    import agentfield_b200 as afb
    from agentfield_b200 import services
    from agentfield_b200.identity import KeySet
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import workflow_cases as WC
    n, K = 1 << 16, 1024
    rng = np.random.default_rng(0xAF2A)
    cache = afb.ExpandedKeys(ctx)
    dids = cache.derive(rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), ["m/44'/%d'/0'" % (8500 + a) for a in range(K)])
    d_exp = torch.from_numpy(cache._expanded).to(dev)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)

    def measure(arrays, nw):
        ki, cols, coff, roff, rcols, rcoff, created = arrays
        D = (t(ki.view(np.int32)), t(cols), t(coff.view(np.int64)), t(roff.view(np.int64)), t(rcols), t(rcoff.view(np.int64)), t(created))
        run = lambda: cache.issue_workflow_dev(*D, nw, d_expanded=d_exp)
        d_docs, d_off, d_pv, d_state, d_summ = run()
        d_st = torch.empty(nw, dtype=torch.uint8, device=dev)
        ks.verify_stored_dev(afb._abi.DOC_WORKFLOW_VC, d_docs, d_off, nw, d_st)
        torch.cuda.synchronize()
        ok = bool((d_state == 0).all()) and bool((d_st == 1).all())
        ms = timed(run)
        ctx.profile_begin()
        timed(run, reps=3)
        kms = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
        m = int(roff[nw])
        return {"workflows": nw, "records": m, "doc_bytes": int(d_off[nw]), "all_verified": ok, "ms": ms, "workflows_per_s": nw / (ms * 1e-3),
                "records_per_s": m / (ms * 1e-3), "kernels_ms": kms}, (d_docs, d_off, d_pv)
    arrays, case = WC.bulk(n, rng, dids, counts=rng.integers(1, 65, n))
    main, (d_docs, d_off, d_pv) = measure(arrays, n)
    # the host-built path on 2000 of the workflows: the same documents, built in Python, signed in one GPU batch
    sample = rng.choice(n, 2000, replace=False)
    svc = services.VCService(cache)
    wfs = []
    for i in sample.tolist():
        c = case(i)
        evs = [{"vc_id": r[0].decode(), "session_id": c["cols"][1].decode(), "status": r[1].decode(), "created_at": WC.time_text(r[2]),
                "issuer_did": c["cols"][2].decode()} for r in c["records"]]
        wfs.append({"workflow_id": c["cols"][0].decode(), "execution_vcs": evs, "root_did": dids[0], "vc_id": c["cols"][3].decode(),
                    "workflow_vc_id": "wvc-%d" % i, "issuance_date": c["cols"][4].decode(), "snapshot_time": c["cols"][5].decode(),
                    "proof_created": c["cols"][6].decode()})
    t_0 = time.perf_counter()
    mirror = svc.generate_workflow_vc_batch(wfs)
    ms_mirror = (time.perf_counter() - t_0) * 1e3
    docs, off = d_docs.cpu().numpy().tobytes(), d_off.cpu().numpy()
    sample_ok = all(m["vc_document"] == docs[int(off[i]):int(off[i + 1])] for m, i in zip(mirror, sample.tolist()))
    mrec = sum(len(w["execution_vcs"]) for w in wfs)
    # the host-buffer call, unpinned arrays
    hdocs, hoff, _, _, _ = cache.issue_workflow_packed(*arrays)
    host_same = hoff[n] == off[n] and hdocs.tobytes() == docs
    t_0 = time.perf_counter()
    for _ in range(3):
        cache.issue_workflow_packed(*arrays)
    ms_host = (time.perf_counter() - t_0) / 3 * 1e3
    del d_docs, d_off, d_pv, hdocs, docs
    torch.cuda.empty_cache()
    # skewed: 1 % of the workflows hold 4096 records
    sk_arrays, _ = WC.bulk(n, rng, dids, counts=rng.integers(1, 65, n), skew=(0.01, 4096))
    skewed, _ = measure(sk_arrays, n)
    ks.close()
    gpu = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return {"gpu": gpu, "dev_call": main, "skewed_1pct_4096": skewed,
            "host_built": {"workflows": len(wfs), "records": mrec, "ms": ms_mirror, "workflows_per_s": len(wfs) / (ms_mirror * 1e-3),
                           "same_documents": bool(sample_ok), "note": "generate_workflow_vc_batch: documents in Python, one GPU signing batch"},
            "host_call": {"workflows": n, "ms": ms_host, "workflows_per_s": n / (ms_host * 1e-3), "same_as_dev": bool(host_same),
                          "note": "unpinned numpy buffers"}}


def register_requests(n, rng, skew=None):
    """2^16-style registration requests: 0-32 reasoners and 0-32 skills with ids like summarize_text_17; 1 % repeat an id, 1 % hold ids
    that need escaping; skew = (fraction, reasoners) gives that fraction of the requests that many reasoners."""
    verbs = [b"summarize", b"translate", b"classify", b"extract", b"rank", b"plan"]
    out = []
    for i in range(n):
        nr, ns = int(rng.integers(0, 33)), int(rng.integers(0, 33))
        if skew and rng.random() < skew[0]:
            nr = skew[1]
        rs = [b"%s_text_%d" % (verbs[k % 6], k) for k in range(nr)]
        ss = [b"%s_skill_%d" % (verbs[(k + 3) % 6], k) for k in range(ns)]
        u = rng.random()
        if u < 0.01 and rs:
            rs.append(rs[0])
        elif u < 0.02 and ss:
            ss[0] = b"tag<\"\xe2\x80\xa8\xff>&"
        out.append({"agent_node_id": b"agent-node-%d" % i, "reasoners": rs, "skills": ss})
    return out


def register_block(ctx, dev, timed):
    """Agent DIDs registered on the device (afc_did_register_batch): 2^16 registrations with 0-32 reasoners and 0-32 skills each (~2.2 M
    components), then a skewed batch in which 1 % of the agents have 1024 reasoners.  Next to it: the same keys through the two calls
    ExpandedKeys.derive makes (SHA-256, then the expansion, on device buffers), the host-buffer call from pinned memory, and the CPU figure:
    the oracle's C port of NewKeyFromSeed over the same seeds on every core."""
    import torch
    import agentfield_b200 as afb
    from oracle import c_oracle as CO
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import did_cases as DC
    n = 1 << 16
    rng = np.random.default_rng(0xAF2B)
    master = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    server = b"agentfield-server-bench"
    cache = afb.ExpandedKeys(ctx)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731

    def measure(reqs):
        nodes, node_off, id_idx, ids, id_off = DC.pack(reqs)
        ai = np.arange(len(reqs), dtype=np.uint32)
        D = (t(np.frombuffer(master, dtype=np.uint8).copy()), server, t(nodes), t(node_off.view(np.int64)), t(ai.view(np.int32)),
             t(id_idx.view(np.int64)), t(ids), t(id_off.view(np.int64)), len(reqs))
        run = lambda: cache.register_dev(*D, append=False)  # noqa: E731
        R = run()
        torch.cuda.synchronize()
        C_ = int(R["comp_off"][-1])
        ms = timed(run)
        ctx.profile_begin()
        timed(run, reps=3)
        kms = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
        return {"registrations": len(reqs), "components": C_, "body_bytes": int(R["body_off"][-1]), "ms": ms,
                "registrations_per_s": len(reqs) / (ms * 1e-3), "components_per_s": C_ / (ms * 1e-3), "kernels_ms": kms}, R, (nodes, node_off, ai, id_idx,
                                                                                                                                  ids, id_off)
    reqs = register_requests(n, rng)
    main, R, arrays = measure(reqs)
    C_ = main["components"]
    # the same keys through today's two calls: SHA-256(master || path), then the expansion
    paths = R["paths"].cpu().numpy()
    plen = (paths != 0).sum(axis=1).astype(np.uint64)
    msgs = np.zeros((C_, 80), dtype=np.uint8)
    msgs[:, :32] = np.frombuffer(master, dtype=np.uint8)
    msgs[:, 32:80] = paths
    flat = np.concatenate([msgs[c, :32 + int(plen[c])] for c in range(C_)])
    off = np.zeros(C_ + 1, dtype=np.uint64)
    off[1:] = np.cumsum(32 + plen)
    d_msgs, d_off = t(flat), t(off.view(np.int64))
    d_seeds = torch.empty((C_, 32), dtype=torch.uint8, device=dev)
    d_exp = torch.empty((C_, 96), dtype=torch.uint8, device=dev)

    def two_calls():
        ctx.sha256_dev(d_msgs, d_off, C_, d_seeds)
        ctx.expand_dev(d_seeds, C_, d_exp)
    two_calls()
    torch.cuda.synchronize()
    same_keys = bool((d_exp == R["expanded"]).all())
    ms_two = timed(two_calls)
    seeds = d_seeds.cpu().numpy()
    del R, d_msgs, d_off, d_exp
    torch.cuda.empty_cache()
    # the host-buffer call from pinned memory
    nodes, node_off, ai, id_idx, ids, id_off = arrays
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()  # noqa: E731
    P = [pin(a) for a in (nodes, node_off, ai, id_idx, ids, id_off)]
    host = lambda: cache.register_packed(master, server, *P, append=False)  # noqa: E731
    host()
    t_0 = time.perf_counter()
    for _ in range(3):
        host()
    ms_host = (time.perf_counter() - t_0) / 3 * 1e3
    # the CPU figure: NewKeyFromSeed (the oracle's C port) on every core, over a 2^16 sample of the seeds
    threads = os.cpu_count() or 1
    cpu_n = min(C_, 1 << 16)
    t_0 = time.perf_counter()
    CO.ed25519_pubkey_batch(np.ascontiguousarray(seeds[:cpu_n]), nthreads=threads)
    s_cpu = time.perf_counter() - t_0
    torch.cuda.empty_cache()
    skewed, _, _ = measure(register_requests(n, rng, skew=(0.01, 1024)))
    gpu = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return {"gpu": gpu, "sign_mode": ctx.sign_mode(), "dev_call": main, "skewed_1pct_1024": skewed,
            "two_calls": {"components": C_, "ms": ms_two, "components_per_s": C_ / (ms_two * 1e-3), "same_keys": same_keys,
                          "note": "sha256_dev + expand_dev: keys only, no DIDs, JWKs or bodies"},
            "host_call": {"registrations": n, "ms": ms_host, "registrations_per_s": n / (ms_host * 1e-3), "components_per_s": C_ / (ms_host * 1e-3),
                          "note": "pinned numpy buffers"},
            "cpu_new_key_from_seed": {"keys": cpu_n, "threads": threads, "s": s_cpu, "keys_per_s": cpu_n / s_cpu}}


def reregister_requests(n, rng, skew=None):
    """A restart storm: n known agents, each with 0-32 registered reasoners and 0-32 skills (as handleNewRegistration stored them, in the
    canonical JWK spelling), re-registering: about 90 % unchanged, 5 % removals only, 5 % partial (new ids, some with removals).
    skew = (fraction, reasoners) gives that fraction of the agents that many registered reasoners."""
    verbs = [b"summarize", b"translate", b"classify", b"extract", b"rank", b"plan"]
    out = []
    for i in range(n):
        nr, ns = int(rng.integers(0, 33)), int(rng.integers(0, 33))
        if skew and rng.random() < skew[0]:
            nr = skew[1]
        agent = {"did": b"did:key:z%046d" % i, "public_key_jwk": b'{"alg":"EdDSA","crv":"Ed25519","kty":"OKP","use":"sig","x":"%043d"}' % i,
                 "derivation_path": b"m/44'/1234567'/%d'" % i}
        for name, cnt, kind, w in (("reasoners", nr, 0, b"text"), ("skills", ns, 1, b"skill")):
            agent[name] = [(b"%s_%s_%d" % (verbs[k % 6], w, k), {"did": b"did:key:z%023d%023d" % (i, k), "public_key_jwk":
                            b'{"alg":"EdDSA","crv":"Ed25519","kty":"OKP","use":"sig","x":"%021d%022d"}' % (i, k),
                            "derivation_path": b"m/44'/1234567'/%d'/%d'/%d'" % (i, kind, k), "function_name": b"%s_%s_%d" % (verbs[k % 6], w, k)})
                           for k in range(cnt)]
        req = {"reasoners": [k for k, _ in agent["reasoners"]], "skills": [k for k, _ in agent["skills"]]}
        u = rng.random()
        if u < 0.05:                                               # removals only
            name = "reasoners" if req["reasoners"] else "skills"
            req[name] = req[name][1:]
        elif u < 0.10:                                             # partial
            req["reasoners"] = req["reasoners"][1:] + [b"new_reasoner_%d" % i]
            req["skills"] = req["skills"] + [b"new_skill_a", b"new_skill_a"]
        out.append({"agent_node_id": b"agent-node-%d" % i, "agent": agent, "reasoners": req["reasoners"], "skills": req["skills"], "agent_index": i})
    return out


def reregister_block(ctx, dev, timed):
    """Known agents re-registered on the device (afc_did_reregister_batch): a restart storm of 2^16 known agents with 0-32 registered
    reasoners and 0-32 skills (about 90 % unchanged, 5 % removals only, 5 % partial), then the same with 1 % of the agents at 1024
    registered reasoners.  Next to it: the host-buffer call from pinned memory, and the oracle (tests/didrr_oracle.py, the
    reference's branch restated in Python on one core) over a sample of the same requests."""
    import torch
    import agentfield_b200 as afb
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import didrr_cases as RC
    n = 1 << 16
    rng = np.random.default_rng(0xAF3C)
    master = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    server = b"agentfield-server-bench"
    cache = afb.ExpandedKeys(ctx)
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).view(dt)).to(dev)  # noqa: E731

    def measure(reqs):
        A = RC.pack(reqs)
        D = (t(np.frombuffer(master, dtype=np.uint8).copy(), np.uint8), server, t(A[0], np.uint8), t(A[1], np.int64), t(A[2], np.int32),
             t(A[3], np.int64), t(A[4], np.uint8), t(A[5], np.int64), t(A[6], np.int64), t(A[7], np.uint8), t(A[8], np.int64), len(reqs))
        run = lambda: cache.reregister_dev(*D, append=False)  # noqa: E731
        R = run()
        torch.cuda.synchronize()
        st = R["state"].cpu().numpy()
        ms = timed(run)
        ctx.profile_begin()
        timed(run, reps=3)
        kms = {k: v["avg_ms"] for k, v in ctx.profile_end().items()}
        return {"agents": len(reqs), "registered_components": int(A[6][-1]), "request_ids": int(A[3][-1]),
                "states": {"unchanged": int((st == 0).sum()), "removed": int((st == 1).sum()), "partial": int((st == 2).sum()),
                           "invalid": int((st == 3).sum())},
                "body_bytes": int(R["body_off"][-1]), "ms": ms, "agents_per_s": len(reqs) / (ms * 1e-3), "kernels_ms": kms}, R, A
    reqs = reregister_requests(n, rng)
    main, R, A = measure(reqs)
    # the host-buffer call from pinned memory
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()  # noqa: E731
    P = [pin(a) for a in A]
    host = lambda: cache.reregister_packed(master, server, P[0], P[1], P[2], *P[3:], append=False)  # noqa: E731
    H = host()
    host_same = bool((H["body"] == R["body"].cpu().numpy()).all() and (H["state"] == R["state"].cpu().numpy()).all())
    t_0 = time.perf_counter()
    for _ in range(3):
        host()
    ms_host = (time.perf_counter() - t_0) / 3 * 1e3
    # the oracle on a sample of the same requests (one core, Python)
    sample = list(range(0, n, 16))
    t_0 = time.perf_counter()
    want = RC.oracle([reqs[i] for i in sample], master=master, server=server)
    s_oracle = time.perf_counter() - t_0
    body = H["body"].tobytes()
    oracle_same = all(body[int(H["body_off"][i]):int(H["body_off"][i + 1])] == w["body"] for i, w in zip(sample, want))
    del R, H, P
    torch.cuda.empty_cache()
    skewed, _, _ = measure(reregister_requests(n, rng, skew=(0.01, 1024)))
    gpu = subprocess.run(["nvidia-smi", "-i", str(dev.index or 0), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return {"gpu": gpu, "sign_mode": ctx.sign_mode(), "dev_call": main, "skewed_1pct_1024": skewed,
            "host_call": {"agents": n, "ms": ms_host, "agents_per_s": n / (ms_host * 1e-3), "same_as_dev": host_same, "note": "pinned numpy buffers"},
            "oracle": {"agents": len(sample), "s": s_oracle, "agents_per_s": len(sample) / s_oracle, "same_bodies": bool(oracle_same),
                       "note": "tests/didrr_oracle.py: the reference's branch restated in Python, one core; not the Go service"}}


def main():
    import torch
    import agentfield_b200 as afb
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", choices=["stored_vc_verify", "audit_stored", "verify_json", "issue_execution", "webhook", "issue_workflow", "register",
                                        "reregister"],
                    default=None,
                    help="run one block")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    ctx = afb.Context(0)

    def timed(fn, reps=args.reps):
        fn(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps
    blocks = {"stored_vc_verify": stored_vc_block, "audit_stored": audit_stored_block, "verify_json": verify_json_block,
              "issue_execution": issue_execution_block, "webhook": webhook_block, "issue_workflow": issue_workflow_block, "register": register_block,
              "reregister": reregister_block}
    print(json.dumps({k: f(ctx, dev, timed) for k, f in blocks.items() if args.only in (None, k)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
