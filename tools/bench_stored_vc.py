#!/usr/bin/env python
"""Stored execution-VC documents verified from their bytes (afc_vc_verify_stored_batch[_dev]) against the keyed-verify floor.
Prints one JSON line: documents/s of the device-pointer call with its per-kernel split, of the keyed verify alone over the same
signing bytes already rendered, and of the host-buffer call; host_fallback and all_expected; the card and its power limit, read
in the same run.  The audit_stored block does the same for the audit of stored execution VCs against their records
(afc_vc_audit_stored_batch[_dev]), next to the stored-verify device call on the same documents.  The verify_json block measures
documents in three client spellings (afc_vc_verify_json_batch_dev) next to the stored-verify call on the canonical form.  Needs a
CUDA device; writes nothing.
usage: python tools/bench_stored_vc.py [--reps R]"""
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


def main():
    import torch
    import agentfield_b200 as afb
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", choices=["stored_vc_verify", "audit_stored", "verify_json"], default=None, help="run one block")
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
    blocks = {"stored_vc_verify": stored_vc_block, "audit_stored": audit_stored_block, "verify_json": verify_json_block}
    print(json.dumps({k: f(ctx, dev, timed) for k, f in blocks.items() if args.only in (None, k)}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
