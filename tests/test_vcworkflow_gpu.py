"""afc_vc_issue_workflow_batch[_dev] on the GPU: documents and proof values equal the OpenSSL-signed oracle (oracle/ref_vc.py) and summaries
the mirror in both signing modes; the host-buffer call equals the _dev call, also with 97-workflow chunks and with a workflow larger than a
staging chunk; every built document verifies under afc_vc_verify_stored_batch(AFC_DOC_WORKFLOW_VC) and audits clean (those holding the U+FFFD escape,
which that verifier leaves to the host, carry a signature over the oracle's signing message); planted HOST cases, empty batches and workflows;
the argument errors; 2^18 workflows of 2^22 records; and VCService.issue_workflow_vc_batch against generate_workflow_vc_batch."""
import base64
import datetime as dt
import os
import subprocess
import sys

import numpy as np
import pytest

import workflow_cases as WC

pytestmark = pytest.mark.gpu

MASTER = bytes(range(32))


def _keys(ctx, k, base=7100):
    import agentfield_b200 as afb
    from oracle import go_hash as H
    cache = afb.ExpandedKeys(ctx)
    paths = ["m/44'/%d'/0'" % (base + a) for a in range(k)]
    dids = cache.derive(MASTER, paths)
    seeds = {d: H.derive_seed(MASTER, p) for d, p in zip(dids, paths)}
    return cache, dids, seeds


def _cases(dids, n, seed, odd=0.15, max_records=12):
    rng = np.random.default_rng(seed)
    return [WC.random_case(rng, i, dids[int(rng.integers(len(dids)))].encode(), max_records=max_records, odd=odd) for i in range(n)]


def _ki(cache, cases):
    return cache.key_index([c["cols"][2].decode() for c in cases])


def _host(cache, cases):
    docs, off, pv, state, summ = cache.issue_workflow_packed(_ki(cache, cases), *WC.pack(cases))
    return docs.tobytes(), off, pv, state, summ


def _dev(ctx, cache, cases):
    import torch
    dev = torch.device("cuda", ctx.device)
    cols, coff, roff, rcols, rcoff, created = WC.pack(cases)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = cache.issue_workflow_dev(t(_ki(cache, cases).view(np.int32)), t(cols), t(coff.view(np.int64)), t(roff.view(np.int64)), t(rcols),
                                   t(rcoff.view(np.int64)), t(created if len(created) else np.zeros(2, dtype=np.int64)), len(cases))
    torch.cuda.synchronize(dev)
    d_docs, d_off, d_pv, d_state, d_summ = out
    return (d_docs.cpu().numpy().tobytes(), d_off.cpu().numpy().astype(np.uint64), d_pv.cpu().numpy(), d_state.cpu().numpy(),
            d_summ.cpu().numpy().view(np.uint32))


def _split(res):
    docs, off, pv, state, summ = res
    return [(docs[int(off[i]):int(off[i + 1])], pv[i].tobytes(), int(state[i]), [int(x) for x in summ[i]]) for i in range(len(state))]


def _check_against_oracle(cases, got, seeds):
    for i, (c, g) in enumerate(zip(cases, got)):
        want = WC.summary(c)
        if want is None:
            assert g == (b"", b"\0" * 86, 1, [0, 0, 0, 0]), i
            continue
        doc, pv = WC.oracle_signed(c, seeds[c["cols"][2].decode()])
        assert g == (doc, pv.encode(), 0, want), (i, g, doc)


@pytest.mark.parametrize("constant_time", [True, False])
def test_equals_oracle(ctx, constant_time):
    cache, dids, seeds = _keys(ctx, 16)
    cases = _cases(dids, 1500, seed=51)
    cases[7]["records"].append((b"vc-x", b"succ\x80eeded", 1_790_000_000, 0))          # planted HOST cases
    cases[8]["records"].append((b"vc-y", b"done", WC.SEC_MAX + 1, 0))
    ctx.sign_configure(constant_time)
    try:
        dev = _split(_dev(ctx, cache, cases))
        host = _split(_host(cache, cases))
    finally:
        ctx.sign_configure(True)
    assert dev == host
    _check_against_oracle(cases, dev, seeds)


def test_built_documents_verify_and_audit_clean(ctx):
    from agentfield_b200 import _abi
    from agentfield_b200.identity import KeySet
    from oracle import go_ed25519 as G, ref_vc as RV
    cache, dids, seeds = _keys(ctx, 12)
    cases = _cases(dids, 1200, seed=52, odd=0.2)
    got = _split(_dev(ctx, cache, cases))
    built = [(c, g) for c, g in zip(cases, got) if g[2] == 0]
    assert len(built) == len(cases)
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    st, _ = ks.verify_stored(_abi.DOC_WORKFLOW_VC, [g[0] for _, g in built])
    ast, iss = ks.audit_stored(_abi.DOC_WORKFLOW_VC, [g[0] for _, g in built])
    n_host = 0
    for (c, g), s, a, m in zip(built, st, ast, iss):
        if b"\\ufffd" in g[0]:
            # an input with invalid UTF-8: json.Unmarshal reads the escape as U+FFFD and json.Marshal writes that rune as it is, so where
            # the escape sits in the signed part, the message verifyWorkflowVCSignature re-marshals differs from the one signed and the
            # reference rejects its own document (in the proof's created it is zeroed before signing).  The stored-document verifier
            # leaves these to the host; the signature holds over the signing message either way.
            assert s == _abi.VC_HOST
            n_host += 1
            pk = cache.public_key(c["cols"][2].decode())
            assert RV.verify_workflow_vc(g[0], pk) == (b"\\ufffd" not in g[0][:g[0].index(b',"proof":')])
            assert G.verify(pk, WC.oracle_docs(c)[0], base64.urlsafe_b64decode(g[1] + b"=="))
        else:
            assert s == _abi.VC_VALID and a == _abi.VC_VALID and m == 0, (s, a, m, g[0])
    assert n_host > 0
    ks.close()


def test_host_and_device_calls_agree(ctx):
    cache, dids, _ = _keys(ctx, 20)
    cases = _cases(dids, 1000, seed=53, max_records=40)
    assert _split(_host(cache, cases)) == _split(_dev(ctx, cache, cases))


def test_chunk_boundaries_in_a_fresh_process():
    """The host-buffer call with chunks of 97 workflows (AFC_CHUNK_ITEMS is read once per process)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, AFC_CHUNK_ITEMS="97", AFC_MIN_CHUNK_ITEMS="97")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(root, "tests", "test_vcworkflow_gpu.py"), "-m", "gpu", "-q", "-x", "-p",
                        "no:cacheprovider", "-k", "test_host_and_device_calls_agree or test_empty_and_planted"],
                       cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "2 passed" in r.stdout, (r.stdout[-2000:], r.stderr[-2000:])


def test_empty_and_planted(ctx):
    from agentfield_b200 import _abi
    cache, dids, seeds = _keys(ctx, 3)
    docs, off, pv, state, summ = _host(cache, [])
    assert off.tolist() == [0] and pv.shape == (0, 86) and state.shape == (0,)
    empty = [{"cols": WC.base_cols(i, dids[i % 3].encode()), "records": []} for i in range(300)]
    got = _split(_host(cache, empty))
    assert got == _split(_dev(ctx, cache, empty))
    _check_against_oracle(empty, got, seeds)
    planted = _cases(dids, 400, seed=54)
    bad = [b"\x00", b"\x1f", b"\x7f", b"\xc3\xa9", "\u212a".encode(), "\u00a0".encode()]     # Kelvin sign, NBSP
    for i, c in enumerate(planted):
        if i % 3 == 0:
            c["records"].insert(0, (b"vc-p", b"done" + bad[i % len(bad)], 1_790_000_000, 0))
        elif i % 3 == 1:
            c["records"].append((b"vc-q", b"ok", [WC.SEC_MIN - 1, WC.SEC_MAX + 1, 0, 0][i % 4], [0, 0, -1, 10 ** 9][i % 4]))
    got = _split(_host(cache, planted))
    assert got == _split(_dev(ctx, cache, planted))
    assert sum(g[2] == _abi.WORKFLOW_HOST for g in got) == sum(1 for i in range(400) if i % 3 != 2)
    _check_against_oracle(planted, got, seeds)


def test_argument_errors(ctx):
    import torch
    from agentfield_b200 import _abi
    lib = _abi.load()
    cache, dids, _ = _keys(ctx, 2)
    cases = _cases(dids, 5, seed=55)
    cases[0]["records"] = cases[0]["records"] or [(b"vc-1", b"done", 1_790_000_000, 0)]
    ki = _ki(cache, cases)
    cols, coff, roff, rcols, rcoff, created = WC.pack(cases)
    exp = cache._expanded
    cap = lib.afc_vc_workflow_bound(_abi.ptr(coff), _abi.ptr(roff), _abi.ptr(rcoff), 5)
    docs, doff = np.empty(cap, dtype=np.uint8), np.zeros(6, dtype=np.uint64)
    pv, st, sm = np.empty((5, 86), dtype=np.uint8), np.empty(5, dtype=np.uint8), np.empty((5, 4), dtype=np.uint32)
    P = _abi.ptr

    def call(**kw):
        a = dict(exp=exp, nk=exp.shape[0], ki=ki, cols=cols, coff=coff, roff=roff, rcols=rcols, rcoff=rcoff, cr=created, docs=docs, cap=cap,
                 doff=doff, pv=pv, st=st, sm=sm, ctx=ctx.handle)
        a.update(kw)
        return lib.afc_vc_issue_workflow_batch(a["ctx"], P(a["exp"]), a["nk"], P(a["ki"]), P(a["cols"]), P(a["coff"]), P(a["roff"]), P(a["rcols"]),
                                               P(a["rcoff"]), P(a["cr"]), 5, P(a["docs"]), a["cap"], P(a["doff"]), P(a["pv"]), P(a["st"]), P(a["sm"]))
    assert call() == _abi.AFC_OK
    assert call(cap=cap - 1) == _abi.AFC_EINVAL
    bad = ki.copy(); bad[3] = exp.shape[0]
    assert call(ki=bad) == _abi.AFC_EINVAL
    assert call(nk=0) == _abi.AFC_EINVAL
    assert call(ctx=None) == _abi.AFC_EINVAL
    for k in ("exp", "ki", "cols", "coff", "roff", "rcols", "rcoff", "cr", "docs", "doff", "pv", "st", "sm"):
        assert call(**{k: None}) == _abi.AFC_EINVAL, k
    back = coff.copy(); back[9] = back[8] - 1 if back[8] else 0; back[8] += 3
    assert call(coff=back) == _abi.AFC_EINVAL
    rb = roff.copy(); rb[2] = rb[3] + 1
    assert call(roff=rb) == _abi.AFC_EINVAL
    rcb = rcoff.copy(); rcb[1] = rcb[2] + 1
    assert call(rcoff=rcb) == _abi.AFC_EINVAL
    dev = torch.device("cuda", ctx.device)
    t = lambda a: torch.from_numpy(a).to(dev)
    d = dict(exp=t(exp), ki=t(ki.view(np.int32)), cols=t(cols), coff=t(coff.view(np.int64)), roff=t(roff.view(np.int64)), rcols=t(rcols),
             rcoff=t(rcoff.view(np.int64)), cr=t(created), docs=torch.empty(cap, dtype=torch.uint8, device=dev),
             doff=torch.empty(6, dtype=torch.int64, device=dev), pv=torch.empty((5, 86), dtype=torch.uint8, device=dev),
             st=torch.empty(5, dtype=torch.uint8, device=dev), sm=torch.empty((5, 4), dtype=torch.int32, device=dev))

    def dcall(cap_, sm_):
        return lib.afc_vc_issue_workflow_batch_dev(ctx.handle, P(d["exp"]), exp.shape[0], P(d["ki"]), P(d["cols"]), P(d["coff"]), P(d["roff"]),
                                                   P(d["rcols"]), P(d["rcoff"]), P(d["cr"]), 5, P(d["docs"]), cap_, P(d["doff"]), P(d["pv"]),
                                                   P(d["st"]), sm_, ctx._stream(None))
    assert dcall(cap, P(d["sm"])) == _abi.AFC_OK
    assert dcall(cap - 1, P(d["sm"])) == _abi.AFC_EINVAL
    assert dcall(cap, None) == _abi.AFC_EINVAL
    torch.cuda.synchronize(dev)


def _service_workflows(dids, n, seed):
    rng = np.random.default_rng(seed)
    base = dt.datetime(2026, 9, 21, 6, 0, 0, tzinfo=dt.timezone.utc)
    out = []
    for i in range(n):
        issuer = dids[int(rng.integers(len(dids)))]
        evs = []
        for j in range(int(rng.integers(0, 10))):
            st = WC.STATUS_SPELLINGS[int(rng.integers(len(WC.STATUS_SPELLINGS)))]
            if i % 17 == 3 and j == 0:
                st = "d\u00f6ne"                                     # not ASCII: this workflow goes through the host path
            t = base + dt.timedelta(seconds=int(rng.integers(0, 30)), microseconds=int(rng.integers(0, 10 ** 6)))
            evs.append({"vc_id": "vc-%d" % (1_790_000_000_000_000_000 + 100 * i + j), "session_id": "sess_%d" % i, "status": st, "created_at": t,
                        "issuer_did": issuer})
        out.append({"workflow_id": "wf_%d" % i, "execution_vcs": evs, "root_did": dids[0], "vc_id": "vc-%d" % (1_790_000_000_000_000_000 + i),
                    "workflow_vc_id": "wvc-%d" % i, "issuance_date": "2026-09-21T06:00:00Z", "snapshot_time": "2026-09-21T06:00:40Z",
                    "proof_created": "2026-09-21T06:00:41Z"})
    return out


def test_service_equals_host_path(ctx):
    from agentfield_b200.services import VCService, _rfc3339
    cache, dids, _ = _keys(ctx, 6)
    wfs = _service_workflows(dids, 300, seed=56)
    svc = VCService(cache)
    got = svc.issue_workflow_vc_batch(wfs)
    text = [dict(w, execution_vcs=[dict(v, created_at=_rfc3339(v["created_at"])) for v in w["execution_vcs"]]) for w in wfs]
    want = svc.generate_workflow_vc_batch(text)
    for w in want:
        del w["doc"], w["proof"]
    assert got == want
    assert svc.issue_workflow_vc_batch([]) == []


def test_large_run(ctx):
    """2^18 workflows and 2^22 records from 1024 issuers: every document verifies on the device and 2000 sampled ones equal the oracle."""
    import torch
    from agentfield_b200 import _abi
    from agentfield_b200.identity import KeySet
    cache, dids, seeds = _keys(ctx, 1024, base=9100)
    n = 1 << 18
    arrays, case = WC.bulk(n, np.random.default_rng(57), dids, max_records=31)
    ki, cols, coff, roff, rcols, rcoff, created = arrays
    m = int(roff[n])
    assert (1 << 22) - (1 << 19) < m < (1 << 22) + (1 << 19)
    dev = torch.device("cuda", ctx.device)
    t = lambda a: torch.from_numpy(a).to(dev)
    d_docs, d_off, d_pv, d_state, d_summ = cache.issue_workflow_dev(t(ki.view(np.int32)), t(cols), t(coff.view(np.int64)), t(roff.view(np.int64)),
                                                                   t(rcols), t(rcoff.view(np.int64)), t(created), n)
    torch.cuda.synchronize(dev)
    assert int((d_state != 0).sum()) == 0
    ks = KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    st = torch.empty(n, dtype=torch.uint8, device=dev)
    ks.verify_stored_dev(_abi.DOC_WORKFLOW_VC, d_docs, d_off, n, st)
    torch.cuda.synchronize(dev)
    assert (st.cpu().numpy() == _abi.VC_VALID).all()
    docs, off, pv, summ = d_docs.cpu().numpy().tobytes(), d_off.cpu().numpy(), d_pv.cpu().numpy(), d_summ.cpu().numpy().view(np.uint32)
    rng = np.random.default_rng(58)
    for i in rng.choice(n, 2000, replace=False).tolist():
        c = case(i)
        doc, p = WC.oracle_signed(c, seeds[c["cols"][2].decode()])
        assert docs[int(off[i]):int(off[i + 1])] == doc and pv[i].tobytes() == p.encode() and summ[i].tolist() == WC.summary(c), i
    ks.close()


def test_skewed_batch_and_a_workflow_larger_than_a_chunk(ctx):
    """1 % of the workflows hold 4096 records; then one workflow of 3.5 M records (more bytes than a staging chunk) between small ones
    in the host-buffer call.  Both calls agree; sampled documents equal the oracle."""
    cache, dids, seeds = _keys(ctx, 64, base=9300)
    n = 1 << 13
    arrays, case = WC.bulk(n, np.random.default_rng(59), dids, max_records=16, skew=(0.01, 4096))
    host = cache.issue_workflow_packed(*arrays)
    dev = _dev_arrays(ctx, cache, arrays, n)
    assert _split((host[0].tobytes(),) + host[1:]) == _split(dev)
    docs, off, pv, _, summ = dev
    for i in list(np.nonzero(np.diff(arrays[3].astype(np.int64)) == 4096)[0][:5]) + [0, 1, n - 1]:
        c = case(int(i))
        doc, p = WC.oracle_signed(c, seeds[c["cols"][2].decode()])
        assert docs[int(off[i]):int(off[i + 1])] == doc and summ[i].tolist() == WC.summary(c)
    arrays, case = WC.bulk(3, np.random.default_rng(61), dids, counts=[5, 3_500_000, 7])
    host = cache.issue_workflow_packed(*arrays)
    dev = _dev_arrays(ctx, cache, arrays, 3)
    assert _split((host[0].tobytes(),) + host[1:]) == _split(dev)
    for i in (0, 2):
        c = case(i)
        doc, _ = WC.oracle_signed(c, seeds[c["cols"][2].decode()])
        assert dev[0][int(dev[1][i]):int(dev[1][i + 1])] == doc
    c = case(1)
    assert dev[4][1].tolist() == WC.summary(c)


def _dev_arrays(ctx, cache, arrays, n):
    import torch
    ki, cols, coff, roff, rcols, rcoff, created = arrays
    dev = torch.device("cuda", ctx.device)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = cache.issue_workflow_dev(t(ki.view(np.int32)), t(cols), t(coff.view(np.int64)), t(roff.view(np.int64)), t(rcols), t(rcoff.view(np.int64)),
                                   t(created if len(created) else np.zeros(2, dtype=np.int64)), n)
    torch.cuda.synchronize(dev)
    d_docs, d_off, d_pv, d_state, d_summ = out
    return (d_docs.cpu().numpy().tobytes(), d_off.cpu().numpy().astype(np.uint64), d_pv.cpu().numpy(), d_state.cpu().numpy(),
            d_summ.cpu().numpy().view(np.uint32))
