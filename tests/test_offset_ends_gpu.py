"""The ends every _dev call reads from its device offset arrays against the host afc_*_bound of the same arrays, for batches that start past
item 0 and record 0: a *_cap equal to the host bound is accepted and one byte less is AFC_EINVAL, and a backwards doc_off / rec_off /
id_idx / reg_idx range is AFC_EINVAL (the stored, JSON and audit calls take no cap: there the batch is accepted and a backwards doc_off
range is not)."""
import random

import numpy as np
import pytest

import did_cases as DC
import didrr_cases as RRC
import resolve_cases as RSC
import workflow_cases as WC
import chain_cases as CC
import test_didresolve_gpu as TR
import test_vcchain_gpu as TC
import test_vcissue_gpu as TI
import test_vcworkflow_gpu as TW
from agentfield_b200 import _abi, services as S

pytestmark = pytest.mark.gpu
P = _abi.ptr


def _dev(ctx):
    import torch
    dev = torch.device("cuda", ctx.device)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a.view(np.int64) if a.dtype == np.uint64 else a)).to(dev)  # noqa: E731
    e = lambda n, dt=None: torch.empty(max(int(n), 1), dtype=dt or torch.uint8, device=dev)  # noqa: E731
    return torch, dev, t, e


def _back(a, stride, k):
    """a (the part of an index array one batch of k items uses) with its last end one below its first"""
    b = np.array(a, dtype=np.uint64)
    b[0] = b[stride * k] + 1
    return b


def _check(ctx, bound, call, backwards):
    """call(cap, **device arrays to replace) runs the _dev call: the host bound is accepted, one byte less and each backwards range are not"""
    import torch
    assert bound > 0
    assert call(bound - 1) == _abi.AFC_EINVAL
    for over in backwards:
        assert call(bound, **over) == _abi.AFC_EINVAL, list(over)
    assert call(bound) == _abi.AFC_OK
    torch.cuda.synchronize(ctx.device)


def _all_verified(status, m):
    """every built document verifies (the batch has no invalid UTF-8, so no document holds the U+FFFD escape)"""
    assert (status == _abi.VC_VALID).all() and len(status) > m // 2, status


def _workflow_batch(ctx, seed):
    cache, dids, _ = TW._keys(ctx, 3, base=7700 + seed)
    cases = TW._cases(dids, 40, seed=seed, odd=0.0)
    for c in cases[:3]:
        c["records"] = c["records"] or [(b"vc-%d" % seed, b"done", 1_790_000_000, 0)]
    return cache, dids, cases


def test_workflow_and_the_calls_over_its_documents(ctx):
    from agentfield_b200.identity import KeySet
    torch, dev, t, e = _dev(ctx)
    lib = _abi.load()
    cache, dids, cases = _workflow_batch(ctx, 1)
    cols, coff, roff, rcols, rcoff, created = WC.pack(cases)
    ki = TW._ki(cache, cases)
    n, i0 = len(cases), 3
    k = n - i0
    exp = t(cache._expanded)
    d = dict(ki=t(ki[i0:].view(np.int32)), cols=t(cols), coff=t(coff[7 * i0:]), roff=t(roff[i0:]), rcols=t(rcols), rcoff=t(rcoff), cr=t(created))
    out = dict(docs=None, doff=e(k + 1, torch.int64), pv=e(k * 86), st=e(k), sm=e(4 * k, torch.int32))
    bound = lib.afc_vc_workflow_bound(P(coff[7 * i0:]), P(roff[i0:]), P(rcoff), k)
    out["docs"] = e(bound)

    def call(cap, **over):
        a = dict(d, **over)
        return lib.afc_vc_issue_workflow_batch_dev(ctx.handle, P(exp), exp.shape[0], P(a["ki"]), P(a["cols"]), P(a["coff"]), P(a["roff"]), P(a["rcols"]),
                                                   P(a["rcoff"]), P(a["cr"]), k, P(out["docs"]), cap, P(out["doff"]), P(out["pv"]), P(out["st"]),
                                                   P(out["sm"]), ctx._stream(None))
    _check(ctx, bound, call, [dict(roff=t(_back(roff[i0:], 1, k)))])

    # the stored, JSON and audit calls over these documents, from document j0 on (absolute offsets into the whole buffer)
    doff = out["doff"].cpu().numpy().view(np.uint64)
    j0 = 5
    m = k - j0
    built = out["st"][:k].cpu().numpy()[j0:] == 0                      # the others are left to the host and have no document
    d_docs, d_off = out["docs"], t(doff[j0:])
    d_back = t(_back(doff[j0:], 1, m))
    ks = KeySet([cache.public_key(x) for x in dids], ctx, dids=dids)
    st, iss = e(m), e(m, torch.int32)
    for f in (lib.afc_vc_verify_stored_batch_dev, lib.afc_vc_verify_json_batch_dev):
        assert f(ctx.handle, ks.handle, _abi.DOC_WORKFLOW_VC, P(d_docs), P(d_back), m, P(st), None, ctx._stream(None)) == _abi.AFC_EINVAL
        assert f(ctx.handle, ks.handle, _abi.DOC_WORKFLOW_VC, P(d_docs), P(d_off), m, P(st), None, ctx._stream(None)) == _abi.AFC_OK
        torch.cuda.synchronize(dev)
        _all_verified(st[:m].cpu().numpy()[built], m)
    audit = lib.afc_vc_audit_stored_batch_dev
    assert audit(ctx.handle, ks.handle, _abi.DOC_WORKFLOW_VC, P(d_docs), P(d_back), None, None, m, P(st), P(iss), ctx._stream(None)) == _abi.AFC_EINVAL
    assert audit(ctx.handle, ks.handle, _abi.DOC_WORKFLOW_VC, P(d_docs), P(d_off), None, None, m, P(st), P(iss), ctx._stream(None)) == _abi.AFC_OK
    torch.cuda.synchronize(dev)
    _all_verified(st[:m].cpu().numpy()[built], m)


def test_issue(ctx):
    torch, dev, t, e = _dev(ctx)
    lib = _abi.load()
    cache, dids, _ = TI._keys(ctx, 3, base=7800)
    reqs = TI._varied_requests(dids, 30, seed=3)
    cols, coff, dur, pay, poff, nil = cache.pack_issue_requests(reqs)
    ki = cache.key_index([r["caller_did"] for r in reqs])
    i0, k = 4, len(reqs) - 4
    exp = t(cache._expanded)
    d = dict(ki=t(ki[i0:].view(np.int32)), cols=t(cols), coff=t(coff[14 * i0:]), dur=t(dur[i0:]), pay=t(pay), poff=t(poff[2 * i0:]), nil=t(nil[2 * i0:]))
    bound = lib.afc_vc_issue_bound(P(coff[14 * i0:]), k)
    out = dict(docs=e(bound), doff=e(k + 1, torch.int64), h=e(k * 86), pv=e(k * 86))

    def call(cap, **over):
        a = dict(d, **over)
        return lib.afc_vc_issue_execution_batch_dev(ctx.handle, P(exp), exp.shape[0], P(a["ki"]), P(a["cols"]), P(a["coff"]), P(a["dur"]), P(a["pay"]),
                                                    P(a["poff"]), P(a["nil"]), _abi.ISSUE_HASH_DATA, k, None, P(out["docs"]), cap, P(out["doff"]),
                                                    P(out["h"]), P(out["pv"]), ctx._stream(None))
    _check(ctx, bound, call, [dict(coff=t(_back(coff[14 * i0:], 14, k)))])


def test_webhook(ctx):
    torch, dev, t, e = _dev(ctx)
    lib = _abi.load()
    import test_webhook_gpu as TH
    cb, co, dur, fl, rb, ro, sb, so = S.pack_webhook_deliveries(TH.random_records(50, seed=9))
    i0, k = 6, 44
    d = dict(co=t(co[8 * i0:]), ro=t(ro[i0:]))
    ins = dict(cb=t(cb), dur=t(dur[i0:]), fl=t(fl[i0:]), rb=t(rb), sb=t(sb), so=t(so[i0:].view(np.int32)))
    bound = lib.afc_webhook_bound(P(co[8 * i0:]), P(ro[i0:]), k)
    out = dict(b=e(bound), off=e(k + 1, torch.int64), h=e(k * 71), st=e(k))

    def call(cap, **over):
        a = dict(d, **over)
        return lib.afc_webhook_sign_batch_dev(ctx.handle, P(ins["cb"]), P(a["co"]), P(ins["dur"]), P(ins["fl"]), P(ins["rb"]), P(a["ro"]), P(ins["sb"]),
                                              P(ins["so"]), k, P(out["b"]), cap, P(out["off"]), P(out["h"]), P(out["st"]), ctx._stream(None))
    _check(ctx, bound, call, [dict(ro=t(_back(ro[i0:], 1, k))), dict(co=t(_back(co[8 * i0:], 8, k)))])


def test_chain(ctx):
    torch, dev, t, e = _dev(ctx)
    lib = _abi.load()
    cache, dids, _, cases, _, directory = TC._setup(ctx, n_random=60, seed=17)
    A = list(CC.pack(cases))
    ki = TC._ki(cache, dids, cases)
    n = len(cases)
    i0 = next(i for i in range(1, n) if A[2][i] > 0)
    k = n - i0
    for j, stride in ((1, 7), (2, 1), (7, 2), (8, 3)):                  # the per-workflow arrays start at workflow i0
        A[j] = A[j][stride * i0:]
    exp = t(cache._expanded)
    d = [t(a) for a in A]
    bound = lib.afc_vc_workflow_chain_bound(P(A[1]), P(A[2]), P(A[4]), P(A[7]), P(A[10]), k)
    out = dict(b=e(bound), off=e(k + 1, torch.int64), st=e(k))
    d_ki = t(ki[i0:].view(np.int32))

    def call(cap, rec_off=None):
        a = list(d)
        if rec_off is not None:
            a[2] = rec_off
        return lib.afc_vc_workflow_chain_batch_dev(ctx.handle, P(exp), exp.shape[0], P(d_ki), *[P(x) for x in a], directory.handle, k, P(out["b"]),
                                                   cap, P(out["off"]), P(out["st"]), ctx._stream(None))
    _check(ctx, bound, call, [dict(rec_off=t(_back(A[2], 1, k)))])


def test_register(ctx):
    import agentfield_b200 as afb
    torch, dev, t, e = _dev(ctx)
    lib = _abi.load()
    keys = afb.ExpandedKeys(ctx)
    reqs = DC.random_requests(random.Random(23), 40, max_ids=6)
    nodes, node_off, id_idx, ids, id_off = DC.pack(reqs)
    i0 = next(i for i in range(1, len(reqs)) if id_idx[2 * i] > 0)
    k = len(reqs) - i0
    ai = np.arange(k, dtype=np.uint32)
    slots = k + int(id_idx[-1] - id_idx[2 * i0])
    master = t(np.frombuffer(DC.MASTER, dtype=np.uint8).copy())
    d = dict(node_off=t(node_off[i0:]), id_idx=t(id_idx[2 * i0:]))
    ins = dict(nodes=t(nodes), ai=t(ai.view(np.int32)), ids=t(ids), id_off=t(id_off))
    bound = lib.afc_did_register_bound(P(node_off[i0:]), P(id_idx[2 * i0:]), P(id_off), k, len(DC.SERVER))
    out = dict(comp=e(k + 1, torch.int64), exp=e(slots * 96), pks=e(slots * 32), dids=e(slots * _abi.DID_CHARS), paths=e(slots * _abi.DID_PATH_SLOT),
               fl=e(slots), body=e(bound), boff=e(k + 1, torch.int64))

    def call(cap, **over):
        a = dict(d, **over)
        return lib.afc_did_register_batch_dev(ctx.handle, P(master), DC.SERVER, len(DC.SERVER), P(ins["nodes"]), P(a["node_off"]), P(ins["ai"]),
                                              P(a["id_idx"]), P(ins["ids"]), P(ins["id_off"]), k, P(out["comp"]), P(out["exp"]), P(out["pks"]),
                                              P(out["dids"]), P(out["paths"]), P(out["fl"]), P(out["body"]), cap, P(out["boff"]), ctx._stream(None))
    _check(ctx, bound, call, [dict(id_idx=t(_back(id_idx[2 * i0:], 2, k)))])


def test_reregister(ctx):
    torch, dev, t, e = _dev(ctx)
    lib = _abi.load()
    reqs = RRC.random_requests(random.Random(29), 40)
    A = list(RRC.pack(reqs))                  # agent_cols, agent_col_off, agent_index, id_idx, ids, id_off, reg_idx, reg_cols, reg_col_off
    n = len(reqs)
    i0 = next(i for i in range(1, n) if A[3][2 * i] > 0 and A[6][2 * i] > 0)
    k = n - i0
    A[1], A[2], A[3], A[6] = A[1][3 * i0:], A[2][i0:], A[3][2 * i0:], A[6][2 * i0:]
    m, G = int(A[3][2 * k] - A[3][0]), int(A[6][2 * k] - A[6][0])
    master = t(np.frombuffer(RRC.MASTER, dtype=np.uint8).copy())
    d = [t(a.view(np.int32) if a.dtype == np.uint32 else a) for a in A]
    bound = lib.afc_did_reregister_bound(P(A[1]), P(A[3]), P(A[5]), P(A[6]), P(A[8]), k, len(RRC.SERVER))
    out = [e(k), e(4 * k, torch.int32), e(2 * k * 96), e(2 * k * 32), e(2 * k * _abi.DID_CHARS), e(2 * k * _abi.DID_PATH_SLOT), e(G), e(m)]
    body, boff = e(bound), e(k + 1, torch.int64)

    def call(cap, id_idx=None, reg_idx=None):
        a = list(d)
        a[3] = a[3] if id_idx is None else id_idx
        a[6] = a[6] if reg_idx is None else reg_idx
        return lib.afc_did_reregister_batch_dev(ctx.handle, P(master), RRC.SERVER, len(RRC.SERVER), *[P(x) for x in a], k, *[P(x) for x in out],
                                                P(body), cap, P(boff), ctx._stream(None))
    _check(ctx, bound, call, [dict(id_idx=t(_back(A[3], 2, k))), dict(reg_idx=t(_back(A[6], 2, k)))])


def test_resolve(ctx):
    torch, dev, t, e = _dev(ctx)
    lib = _abi.load()
    reg = RSC.fixture_registry()
    directory = TR.directory_of(ctx, reg)
    kinds, reqs, off = directory.pack_requests(RSC.random_requests(reg, np.random.default_rng(31), 60))
    i0, k = 7, 53
    d_kinds, d_reqs, d_off = t(kinds[i0:]), t(reqs), t(off[i0:])
    bound = lib.afc_did_resolve_bound(directory.handle, P(off[i0:]), k)
    out = dict(b=e(bound), off=e(k + 1, torch.int64), st=e(k))

    def call(cap, req_off=d_off):
        return lib.afc_did_resolve_batch_dev(ctx.handle, directory.handle, P(d_kinds), P(d_reqs), P(req_off), k, P(out["b"]), cap, P(out["off"]),
                                             P(out["st"]), ctx._stream(None))
    _check(ctx, bound, call, [dict(req_off=t(_back(off[i0:], 1, k)))])
