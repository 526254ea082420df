"""The host-buffer and _dev forms of each service call against each other.

(a) Every condition either form checks gives the same return code in both: each required NULL pointer, a capacity one byte below the
    bound, and each count limit that offsets alone reach.  A host form over a count limit runs in a child process, so that a check made
    after the inner array it guards is read fails this test instead of the session; a _dev form is never given an over-limit count.
(b) One batch (one chunk of the host form) launches the same kernels, as many times, in both forms, once the fixed-base table is built;
    only the _dev forms read their offset ends on the device (k_offset_ends, k_dres_ends).
"""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import chain_cases as CC
import did_cases as DC
import didrr_cases as RRC
import resolve_cases as RSC
import workflow_cases as WC
import test_didresolve_gpu as TR
import test_vcchain_gpu as TC
import test_vcissue_gpu as TI
import test_vcworkflow_gpu as TW
from agentfield_b200 import _abi, services as S

pytestmark = pytest.mark.gpu
P = _abi.ptr
EINVAL, ESTATE = _abi.AFC_EINVAL, _abi.AFC_ESTATE
ENDS_KERNELS = ("k_offset_ends", "k_dres_ends")


class Call:
    """One service call: its arguments by name, in ABI order, with numpy arrays for buffers (copied to the device for the _dev form;
    bytes stay host memory in both forms), the capacity argument and its bound, and the pointers it needs for this batch"""

    def __init__(self, fn, args, required, cap=None, bound=None):
        self.fn, self.args, self.required, self.cap, self.bound = fn, args, required, cap, bound

    def run(self, lib, c, dev, **over):
        a = dict(self.args, **over)
        if not dev:
            return getattr(lib, self.fn)(*[P(v) if isinstance(v, np.ndarray) else v for v in a.values()])
        import torch
        keep = []

        def d(v):
            if not isinstance(v, np.ndarray):
                return v
            v = v.view(np.int64) if v.dtype == np.uint64 else v.view(np.int32) if v.dtype == np.uint32 else v
            dev = torch.device("cuda", c.device)
            keep.append(torch.from_numpy(np.ascontiguousarray(v)).to(dev) if v.size else torch.empty(16, dtype=torch.uint8, device=dev))
            return P(keep[-1])
        rc = getattr(lib, self.fn + "_dev")(*[d(v) for v in a.values()], c._stream(None))
        torch.cuda.synchronize(c.device)
        return rc


def _u8(n):
    return np.zeros(max(int(n), 1), dtype=np.uint8)


def _workflow(ctx):
    cache, dids, _ = TW._keys(ctx, 3, base=8100)
    cases = TW._cases(dids, 40, seed=5, odd=0.0)
    for c in cases[:3]:
        c["records"] = c["records"] or [(b"vc-forms", b"done", 1_790_000_000, 0)]
    cols, coff, roff, rcols, rcoff, created = WC.pack(cases)
    n = len(cases)
    lib = _abi.load()
    bound = lib.afc_vc_workflow_bound(P(coff), P(roff), P(rcoff), n)
    args = dict(ctx=ctx.handle, exp=cache._expanded, n_keys=cache._expanded.shape[0], ki=TW._ki(cache, cases), cols=cols, coff=coff, roff=roff,
                rcols=rcols, rcoff=rcoff, created=created, n=n, docs=_u8(bound), cap=bound, doff=np.zeros(n + 1, np.uint64), pv=_u8(86 * n),
                st=_u8(n), sm=np.zeros(4 * n, np.uint32))
    return cache, dids, Call("afc_vc_issue_workflow_batch", args, [k for k in args if k not in ("n_keys", "n", "cap")], "cap", bound)


def _stored(ctx, wf, fn, named=True):
    """stored, JSON or audit over the workflow documents (the audit without columns, as workflow documents take none)"""
    from agentfield_b200.identity import KeySet
    cache, dids, call = wf
    lib = _abi.load()
    assert call.run(lib, ctx, False) == 0
    docs, doff, n = call.args["docs"], call.args["doff"], call.args["n"]
    ks = KeySet([cache.public_key(x) for x in dids], ctx, dids=dids) if named else KeySet([cache.public_key(x) for x in dids], ctx)
    args = dict(ctx=ctx.handle, ks=ks.handle, kind=_abi.DOC_WORKFLOW_VC, docs=docs, doff=doff.copy())
    if fn == "afc_vc_audit_stored_batch":
        args.update(cols=None, coff=None, n=n, st=_u8(n), issues=np.zeros(n, np.uint32))
    else:
        args.update(n=n, st=_u8(n), fields=np.zeros(4 * n, np.uint32))
    c = Call(fn, args, [k for k in ("ctx", "ks", "docs", "doff", "st", "issues") if k in args])
    c.keyset = ks
    return c


def _verify_requests(ctx, wf):
    from agentfield_b200.crypto import pack
    from agentfield_b200.identity import KeySet
    cache, dids, call = wf
    lib = _abi.load()
    assert call.run(lib, ctx, False) == 0
    docs, doff = call.args["docs"], call.args["doff"]
    bodies = [b'{"vc_document":' + bytes(docs[doff[i]:doff[i + 1]]) + b"}" for i in range(call.args["n"])]
    reqs, roff = pack(bodies)
    n = len(bodies)
    ks = KeySet([cache.public_key(x) for x in dids], ctx, dids=dids)
    bound = lib.afc_vc_verify_request_bound(P(roff), n)
    args = dict(ctx=ctx.handle, ks=ks.handle, reqs=reqs, roff=roff, n=n, bodies=_u8(bound), cap=bound, boff=np.zeros(n + 1, np.uint64), st=_u8(n))
    c = Call("afc_vc_verify_request_batch", args, ["ctx", "ks", "reqs", "roff", "bodies", "boff", "st"], "cap", bound)
    c.keyset = ks
    return c


def _issue(ctx):
    cache, dids, _ = TI._keys(ctx, 3, base=8200)
    reqs = TI._varied_requests(dids, 30, seed=4)
    cols, coff, dur, pay, poff, nil = cache.pack_issue_requests(reqs)
    n = len(reqs)
    bound = _abi.load().afc_vc_issue_bound(P(coff), n)
    args = dict(ctx=ctx.handle, exp=cache._expanded, n_keys=cache._expanded.shape[0], ki=cache.key_index([r["caller_did"] for r in reqs]), cols=cols,
                coff=coff, dur=dur, pay=pay, poff=poff, nil=nil, flags=_abi.ISSUE_HASH_DATA, n=n, log=None, docs=_u8(bound), cap=bound,
                doff=np.zeros(n + 1, np.uint64), h=_u8(86 * n), pv=_u8(86 * n))
    return Call("afc_vc_issue_execution_batch", args, [k for k in args if k not in ("n_keys", "flags", "n", "log", "cap")], "cap", bound)


def _chain(ctx):
    cache, dids, _, cases, _, directory = TC._setup(ctx, n_random=40, seed=19)
    A = CC.pack(cases)
    n = len(cases)
    assert A[2][n] > A[2][0]
    bound = _abi.load().afc_vc_workflow_chain_bound(P(A[1]), P(A[2]), P(A[4]), P(A[7]), P(A[10]), n)
    args = dict(ctx=ctx.handle, exp=cache._expanded, n_keys=cache._expanded.shape[0], ki=TC._ki(cache, dids, cases))
    args.update(("a%d" % j, a) for j, a in enumerate(A))
    args.update(dir=directory.handle, n=n, bodies=_u8(bound), cap=bound, boff=np.zeros(n + 1, np.uint64), st=_u8(n))
    c = Call("afc_vc_workflow_chain_batch", args, [k for k in args if k not in ("n_keys", "n", "cap")], "cap", bound)
    c.directory = directory
    return c


def _resolve(ctx):
    reg = RSC.fixture_registry()
    directory = TR.directory_of(ctx, reg)
    kinds, reqs, off = directory.pack_requests(RSC.random_requests(reg, np.random.default_rng(37), 60))
    n = len(off) - 1
    bound = _abi.load().afc_did_resolve_bound(directory.handle, P(off), n)
    args = dict(ctx=ctx.handle, dir=directory.handle, kinds=kinds, reqs=reqs, roff=off, n=n, bodies=_u8(bound), cap=bound,
                boff=np.zeros(n + 1, np.uint64), st=_u8(n))
    c = Call("afc_did_resolve_batch", args, ["ctx", "dir", "kinds", "reqs", "roff", "bodies", "boff", "st"], "cap", bound)
    c.directory = directory
    return c


def _webhook(ctx):
    import test_webhook_gpu as TH
    cb, co, dur, fl, rb, ro, sb, so = S.pack_webhook_deliveries(TH.random_records(50, seed=11))
    n = len(dur)
    assert ro[n] > ro[0] and so[n] > so[0]
    bound = _abi.load().afc_webhook_bound(P(co), P(ro), n)
    args = dict(ctx=ctx.handle, cb=cb, co=co, dur=dur, fl=fl, rb=rb, ro=ro, sb=sb, so=so, n=n, bodies=_u8(bound), cap=bound,
                boff=np.zeros(n + 1, np.uint64), h=_u8(71 * n), st=_u8(n))
    return Call("afc_webhook_sign_batch", args, [k for k in args if k not in ("n", "cap")], "cap", bound)


def _register(ctx):
    reqs = DC.random_requests(random.Random(41), 40, max_ids=6)
    nodes, node_off, id_idx, ids, id_off = DC.pack(reqs)
    n = len(reqs)
    slots = n + int(id_idx[-1] - id_idx[0])
    assert id_off[-1] > id_off[0]
    bound = _abi.load().afc_did_register_bound(P(node_off), P(id_idx), P(id_off), n, len(DC.SERVER))
    args = dict(ctx=ctx.handle, master=np.frombuffer(DC.MASTER, dtype=np.uint8).copy(), server=DC.SERVER, server_len=len(DC.SERVER), nodes=nodes,
                node_off=node_off, ai=np.arange(n, dtype=np.uint32), id_idx=id_idx, ids=ids, id_off=id_off, n=n, comp=np.zeros(n + 1, np.uint64),
                exp=_u8(slots * 96), pks=_u8(slots * 32), dids=_u8(slots * _abi.DID_CHARS), paths=_u8(slots * _abi.DID_PATH_SLOT),
                fl=_u8(slots), body=_u8(bound), cap=bound, boff=np.zeros(n + 1, np.uint64))
    return Call("afc_did_register_batch", args, [k for k in args if k not in ("server_len", "n", "cap")], "cap", bound)


def _reregister(ctx):
    reqs = RRC.random_requests(random.Random(43), 40)
    A = RRC.pack(reqs)                  # agent_cols, agent_col_off, agent_index, id_idx, ids, id_off, reg_idx, reg_cols, reg_col_off
    n = len(reqs)
    m, G = int(A[3][2 * n] - A[3][0]), int(A[6][2 * n] - A[6][0])
    assert m and G and A[5][-1] > A[5][0] and A[8][-1] > A[8][0]
    bound = _abi.load().afc_did_reregister_bound(P(A[1]), P(A[3]), P(A[5]), P(A[6]), P(A[8]), n, len(RRC.SERVER))
    args = dict(ctx=ctx.handle, master=np.frombuffer(RRC.MASTER, dtype=np.uint8).copy(), server=RRC.SERVER, server_len=len(RRC.SERVER))
    args.update(zip(("acols", "acoff", "ai", "id_idx", "ids", "id_off", "reg_idx", "rcols", "rcoff"), A))
    args.update(n=n, st=_u8(n), counts=np.zeros(4 * n, np.uint32), exp=_u8(2 * n * 96), pks=_u8(2 * n * 32), dids=_u8(2 * n * _abi.DID_CHARS),
                paths=_u8(2 * n * _abi.DID_PATH_SLOT), rfl=_u8(G), ifl=_u8(m), body=_u8(bound), cap=bound, boff=np.zeros(n + 1, np.uint64))
    return Call("afc_did_reregister_batch", args, [k for k in args if k not in ("server_len", "n", "cap")], "cap", bound)


@pytest.fixture(scope="module")
def calls(ctx):
    wf = _workflow(ctx)
    return {"_workflow": wf, "stored": _stored(ctx, wf, "afc_vc_verify_stored_batch"), "json": _stored(ctx, wf, "afc_vc_verify_json_batch"),
            "audit": _stored(ctx, wf, "afc_vc_audit_stored_batch"), "verify_request": _verify_requests(ctx, wf), "issue": _issue(ctx),
            "workflow": wf[2], "chain": _chain(ctx), "resolve": _resolve(ctx), "webhook": _webhook(ctx), "register": _register(ctx),
            "reregister": _reregister(ctx)}


NAMES = ["stored", "json", "audit", "verify_request", "issue", "workflow", "chain", "resolve", "webhook", "register", "reregister"]


def _both(lib, c, call, **over):
    return call.run(lib, c, False, **over), call.run(lib, c, True, **over)


@pytest.mark.parametrize("name", NAMES)
def test_rejections(ctx, calls, name):
    lib = _abi.load()
    call = calls[name]
    for arg in call.required:
        assert _both(lib, ctx, call, **{arg: None}) == (EINVAL, EINVAL), arg
    if call.cap:
        assert _both(lib, ctx, call, **{call.cap: call.bound - 1}) == (EINVAL, EINVAL)
        assert _both(lib, ctx, call) == (0, 0)


def test_rejections_of_the_stored_calls_beyond_pointers(ctx, calls):
    lib = _abi.load()
    for name in ("stored", "json", "audit"):
        call = calls[name]
        assert _both(lib, ctx, call, kind=7) == (EINVAL, EINVAL), name
        plain = _stored(ctx, calls["_workflow"], call.fn, named=False)
        assert _both(lib, ctx, plain) == (ESTATE, ESTATE), name
        if name == "audit":                 # the audit's own argument errors win over a keyset without DIDs
            assert _both(lib, ctx, plain, issues=None) == (EINVAL, EINVAL)
            assert _both(lib, ctx, plain, cols=_u8(4), coff=np.zeros(11, np.uint64)) == (EINVAL, EINVAL)
            assert _both(lib, ctx, call, kind=_abi.DOC_EXECUTION_VC) == (EINVAL, EINVAL)          # execution documents need columns
    issue = calls["issue"]
    assert _both(lib, ctx, issue, n_keys=0) == (EINVAL, EINVAL)
    assert _both(lib, ctx, issue, flags=_abi.ISSUE_HASH_DATA | 0x100) == (EINVAL, EINVAL)


def test_request_byte_limit_on_the_device(ctx, calls):
    """a request of 2^31 bytes: the _dev form reads only the offsets (k_dres_ends), so it is given one"""
    lib = _abi.load()
    for name in ("verify_request", "resolve"):
        call = calls[name]
        off = call.args["roff"].copy()
        off[1:] += 1 << 31
        assert call.run(lib, ctx, True, roff=off) == EINVAL, name


_CHILD = r"""
import json
import numpy as np
import agentfield_b200 as afb
import resolve_cases as RSC
import test_didresolve_gpu as TR
import test_vcworkflow_gpu as TW
from agentfield_b200 import _abi
from agentfield_b200.identity import KeySet
ctx = afb.Context(0)
lib = _abi.load()
directory = TR.directory_of(ctx, RSC.fixture_registry())
cache, dids, _ = TW._keys(ctx, 1, base=8300)
keyset = KeySet([cache.public_key(dids[0])], ctx, dids=dids)
keep = []
def arr(a):
    keep.append(a)
    return _abi.ptr(a)
u64 = lambda *v: arr(np.array(v, dtype=np.uint64))
z = lambda k, dt=np.uint8: arr(np.zeros(k, dtype=dt))
keys, ki, cap, big = z(2 * 96), z(1, np.uint32), 1 << 40, 1 << 31
rc = {}
# one request of 2^31 bytes: nothing but its offsets is read
rc["resolve"] = lib.afc_did_resolve_batch(ctx.handle, directory.handle, z(1), z(1), u64(0, big), 1, z(64), cap, z(2, np.uint64), z(1))
rc["verify_request"] = lib.afc_vc_verify_request_batch(ctx.handle, keyset.handle, z(1), u64(0, big), 1, z(64), cap, z(2, np.uint64), z(1))
# a workflow of 2^32 records: rec_col_off (one word here) is not read
rc["workflow"] = lib.afc_vc_issue_workflow_batch(ctx.handle, keys, 2, ki, z(8), z(8, np.uint64), u64(0, 1 << 32), z(8), z(1, np.uint64),
                                                 z(2, np.int64), 1, z(64), cap, z(2, np.uint64), z(86), z(1), z(4, np.uint32))
# 2^31 records in a chain: vcc_slots_fit rejects them before rec_col_off and chain_rec_col_off (one word each here) are read
rc["chain"] = lib.afc_vc_workflow_chain_batch(ctx.handle, keys, 2, ki, z(8), z(8, np.uint64), u64(0, big), z(8), z(1, np.uint64), z(2, np.int64),
                                              z(8), z(3, np.uint64), z(3, np.int64), z(8), z(1, np.uint64), z(1), z(1, np.int64), z(1, np.int32),
                                              directory.handle, 1, z(64), cap, z(2, np.uint64), z(1))
# 2^32 - 1 ids for one request (m + n over 2^32 - 1), before id_off (one word here) is read
rc["register"] = lib.afc_did_register_batch(ctx.handle, z(32), b"s", 1, z(1), u64(0, 1), z(1, np.uint32), u64(0, 0, (1 << 32) - 1), z(1),
                                            z(1, np.uint64), 1, z(2, np.uint64), z(96), z(32), z(64), z(64), z(1), z(64), cap, z(2, np.uint64))
# ids or components over 2^32 - 1 - 2 n, before id_off and reg_col_off (one word each here) are read
def rereg(ids, regs):
    return lib.afc_did_reregister_batch(ctx.handle, z(32), b"s", 1, z(8), z(4, np.uint64), z(1, np.uint32), u64(0, 0, ids), z(1),
                                        z(1, np.uint64), u64(0, 0, regs), z(1), z(1, np.uint64), 1, z(1), z(4, np.uint32), z(192), z(64),
                                        z(128), z(128), z(1), z(1), z(64), cap, z(2, np.uint64))
rc["reregister_ids"] = rereg((1 << 32) - 2, 0)
rc["reregister_components"] = rereg(0, (1 << 32) - 2)
print(json.dumps(rc))
"""


def test_count_limits_of_the_host_forms():
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    out = subprocess.run([sys.executable, "-c", _CHILD], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    rc = json.loads(out.stdout.strip().splitlines()[-1])
    assert rc == {k: EINVAL for k in rc} and len(rc) == 7, rc


def _kernels(ctx, run):
    ctx.profile_begin()
    assert run() == 0
    prof = ctx.profile_end()
    return {k: v["count"] for k, v in prof.items() if k not in ENDS_KERNELS}


@pytest.mark.parametrize("name", NAMES)
def test_same_kernels(ctx, calls, name):
    lib = _abi.load()
    call = calls[name]
    assert call.args["n"] < 65536
    assert _both(lib, ctx, call) == (0, 0)              # warm-up: the fixed-base table is built once per context
    host = _kernels(ctx, lambda: call.run(lib, ctx, False))
    dev = _kernels(ctx, lambda: call.run(lib, ctx, True))
    assert host and host == dev, (host, dev)
