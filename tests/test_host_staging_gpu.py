"""The staging pipeline every host-buffer call runs through: each call gives byte-identical results with all caller buffers pageable, all
pinned and alternating, equal to its _dev call, in 97-item chunks that wrap the slot ring several times; and no seed, webhook secret,
expanded-key half or private JWK stays behind in the context's staging memory after the calls that handle them."""
import base64
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASTER = bytes(range(0x40, 0x60))              # DID registration's master seed
ISSUERS = bytes(range(0x20))                    # the master seed the issuers' keys are derived from (derive hashes it in the clear)
N = 1000


class In:
    """An input buffer: pageable or pinned in a host call, copied to the device for the _dev call."""
    def __init__(self, a):
        self.a = np.ascontiguousarray(a)


class Out(In):
    """An output buffer: zeroed before each call and compared afterwards."""


class Host:
    """A host value that the _dev call also takes from host memory."""
    def __init__(self, a):
        self.a = a


def pinned_like(lib, a):
    """A pinned host copy of numpy array a, allocated through the library (afc_alloc_pinned)."""
    nbytes = a.nbytes
    p = lib.afc_alloc_pinned(max(nbytes, 1))
    if not p:
        raise MemoryError("afc_alloc_pinned(%d)" % nbytes)
    h = np.frombuffer((C.c_uint8 * max(nbytes, 1)).from_address(p), dtype=np.uint8)[:nbytes].view(a.dtype).reshape(a.shape)
    h[...] = a
    return h, p


def host_call(lib, ctx, fn, args, mode):
    """fn(ctx, *args) with caller buffers pageable, pinned or alternating (mode); returns the outputs as uint8 arrays."""
    from agentfield_b200 import _abi
    bufs, keep, outs, pins = [], [], [], []
    for x in args:
        if isinstance(x, (In, Out)):
            a = np.zeros_like(x.a) if isinstance(x, Out) else x.a.copy()
            if mode == "pinned" or (mode == "mixed" and len(keep) % 2 == 0):
                a, p = pinned_like(lib, a)
                pins.append(p)
            keep.append(a)
            if isinstance(x, Out):
                outs.append(a)
            bufs.append(_abi.ptr(a))
        else:
            bufs.append(x.a if isinstance(x, Host) else x)
    try:
        _abi.check(getattr(lib, fn)(ctx.handle, *bufs), ctx.handle)
        return [o.view(np.uint8).reshape(-1).copy() for o in outs]
    finally:
        for p in pins:
            lib.afc_free_pinned(p)


def dev_call(lib, ctx, fn, args):
    import torch
    from agentfield_b200 import _abi
    dev = torch.device("cuda", ctx.device)
    bufs, keep, outs = [], [], []
    for x in args:
        if isinstance(x, Out):
            t = torch.zeros(max(x.a.nbytes, 1), dtype=torch.uint8, device=dev)
            outs.append((t, x.a.nbytes))
            bufs.append(_abi.ptr(t))
        elif isinstance(x, In):
            t = torch.from_numpy(x.a.view(np.uint8).reshape(-1).copy()).to(dev) if x.a.nbytes else None
            keep.append(t)
            bufs.append(_abi.ptr(t))
        else:
            bufs.append(x.a if isinstance(x, Host) else x)
    _abi.check(getattr(lib, fn)(ctx.handle, *bufs, None), ctx.handle)
    torch.cuda.synchronize(dev)
    return [t.cpu().numpy()[:nb] for t, nb in outs]


def packed(rng, n, lo, hi, dtype=np.uint64):
    lens = rng.integers(lo, hi + 1, n)
    off = np.zeros(n + 1, dtype=dtype)
    off[1:] = np.cumsum(lens).astype(dtype)
    return rng.integers(0, 256, int(off[-1]) + 8, dtype=np.uint8), off


def cases(ctx, log_for):
    """(name, host function, its arguments, _dev function, its arguments) for every host-buffer call (None for the _dev function: the
    host function's name with _dev, called with the host function's arguments), and what the secrets test needs besides.  log_for stands
    for the log of the issue call that appends to one."""
    import agentfield_b200 as afb
    import did_cases as DC
    import workflow_cases as WC
    from agentfield_b200 import _abi, canonical as CA, services as S
    rng = np.random.default_rng(0x57A6)
    out = []
    msgs, off = packed(rng, N, 0, 300)
    keys, koff = packed(rng, N, 0, 90, np.uint32)
    out.append(("sha256", "afc_sha256_batch", [In(msgs), In(off), N, Out(np.zeros((N, 32), np.uint8))], None, None))
    out.append(("hmac", "afc_hmac_sha256_batch", [In(keys), In(koff), In(msgs), In(off), N, Out(np.zeros((N, 32), np.uint8))], None, None))
    seeds = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    pks = ctx.pubkeys(seeds)
    sigs = ctx.sign_packed(seeds, msgs, off)
    sigs[::7, 5] ^= 1
    out.append(("pubkey", "afc_ed25519_pubkey_batch", [In(seeds), N, Out(np.zeros((N, 32), np.uint8))], None, None))
    out.append(("expand", "afc_ed25519_expand_batch", [In(seeds), N, Out(np.zeros((N, 96), np.uint8))], None, None))
    out.append(("verify", "afc_ed25519_verify_batch", [In(pks), In(sigs), In(msgs), In(off), N, Out(np.zeros(N, np.uint8))], None, None))
    out.append(("sign", "afc_ed25519_sign_batch", [In(seeds), In(msgs), In(off), N, Out(np.zeros((N, 64), np.uint8))], None, None))
    exp = ctx.expand(seeds)
    ki = rng.integers(0, 13, N).astype(np.uint32)
    out.append(("sign_expanded_key_index", "afc_ed25519_sign_expanded_batch", [In(exp[:13]), In(ki), 13, In(msgs), In(off), N, Out(np.zeros((N, 64), np.uint8))],
                "afc_ed25519_sign_expanded_keys_batch_dev", [In(exp[:13]), 13, In(ki), In(msgs), In(off), N, Out(np.zeros((N, 64), np.uint8))]))
    out.append(("sign_expanded", "afc_ed25519_sign_expanded_batch", [In(exp), None, N, In(msgs), In(off), N, Out(np.zeros((N, 64), np.uint8))],
                "afc_ed25519_sign_expanded_keys_batch_dev", [In(exp), N, None, In(msgs), In(off), N, Out(np.zeros((N, 64), np.uint8))]))
    ks = afb.KeySet([bytes(p) for p in pks[:13]], ctx)
    kv_sigs = ctx.sign_packed(seeds[ki], msgs, off)
    kv_sigs[::5, 9] ^= 4
    out.append(("verify_keyed", "afc_ed25519_verify_keyed_batch", [ks.handle, In(ki), In(kv_sigs), In(msgs), In(off), N, Out(np.zeros(N, np.uint8))],
                None, None))
    # stored documents, signed by derived keys whose DIDs the named keyset resolves
    cache = afb.ExpandedKeys(ctx)
    dids = cache.derive(ISSUERS, ["m/44'/%d'/0'" % (7300 + a) for a in range(11)])
    import torch
    dev = torch.device("cuda", ctx.device)
    d_ki = torch.from_numpy(rng.integers(0, 11, N).astype(np.int32)).to(dev)
    d_docs, d_doff, _, _, _, d_cols, d_coff = CA.synthetic_stored_vcs_dev(ctx, torch.from_numpy(cache._expanded).to(dev), dids, d_ki, N, seed=3,
                                                                          audit_columns=True)
    docs, doff = d_docs.cpu().numpy(), d_doff.cpu().numpy().view(np.uint64)
    cols, coff = d_cols.cpu().numpy(), d_coff.cpu().numpy().view(np.uint64)
    docs[int(doff[17]) + 200] ^= 1                                          # one document that no longer verifies
    cols[int(coff[23 * 10 + 2])] ^= 1                                       # one record that no longer matches its document
    nks = afb.KeySet([cache.public_key(d) for d in dids], ctx, dids=dids)
    for name, fn in (("stored", "afc_vc_verify_stored_batch"), ("json", "afc_vc_verify_json_batch")):
        out.append((name, fn, [nks.handle, _abi.DOC_EXECUTION_VC, In(docs), In(doff), N, Out(np.zeros(N, np.uint8)), Out(np.zeros((N, 4), np.uint32))],
                    None, None))
    out.append(("audit", "afc_vc_audit_stored_batch", [nks.handle, _abi.DOC_EXECUTION_VC, In(docs), In(doff), In(cols), In(coff), N,
                                                       Out(np.zeros(N, np.uint8)), Out(np.zeros(N, np.uint32))], None, None))
    # issue, with hashing on and off, and with a log
    reqs = CA.synthetic_issue_requests(dids, N, seed=5, payload_bytes=(0, 700), nil_frac=0.1, err_frac=0.2)
    ikey = cache.key_index([r["caller_did"] for r in reqs])
    icols, icoff, idur, ipay, ipoff, inil = cache.pack_issue_requests(reqs)
    cap = int(_abi.load().afc_vc_issue_bound(_abi.ptr(icoff), N))
    for name, flags, log in (("issue", _abi.ISSUE_HASH_DATA, False), ("issue_no_hash", 0, False), ("issue_log", _abi.ISSUE_HASH_DATA, True)):
        args = [In(cache._expanded), cache._expanded.shape[0], In(ikey), In(icols), In(icoff), In(idur), In(ipay), In(ipoff), In(inil), flags, N,
                log_for if log else None, Out(np.zeros(cap, np.uint8)), cap, Out(np.zeros(N + 1, np.uint64)),
                Out(np.zeros((N, 86), np.uint8)) if flags else None, Out(np.zeros((N, 86), np.uint8))]
        out.append((name, "afc_vc_issue_execution_batch", args, None, None))
    # workflows
    wcases = [WC.random_case(rng, i, dids[int(rng.integers(len(dids)))].encode(), max_records=12, odd=0.15) for i in range(N)]
    wkey = cache.key_index([c["cols"][2].decode() for c in wcases])
    wcols, wcoff, wroff, wrcols, wrcoff, wcreated = WC.pack(wcases)
    cap = int(_abi.load().afc_vc_workflow_bound(_abi.ptr(wcoff), _abi.ptr(wroff), _abi.ptr(wrcoff), N))
    out.append(("workflow", "afc_vc_issue_workflow_batch",
                [In(cache._expanded), cache._expanded.shape[0], In(wkey), In(wcols), In(wcoff), In(wroff), In(wrcols), In(wrcoff), In(wcreated), N,
                 Out(np.zeros(cap, np.uint8)), cap, Out(np.zeros(N + 1, np.uint64)), Out(np.zeros((N, 86), np.uint8)), Out(np.zeros(N, np.uint8)),
                 Out(np.zeros((N, 4), np.uint32))], None, None))
    # webhook deliveries
    prng = random.Random(7)
    recs = [dict(execution_id="exec_%d" % i, run_id="run_%d" % (i % 3), status=prng.choice(["succeeded", "failed", "DONE"]), node_id="node",
                 reasoner_id="fn_%d" % (i % 7), target_type="reasoner", timestamp="2026-09-21T06:30:%02dZ" % (i % 60),
                 duration_ms=prng.choice([None, 5, -2 ** 63]), result=prng.choice([b'{"b":2,"a":[1,2.5]}', b"null", b"", b'"x\\u00e9"']),
                 error_message=prng.choice([None, "boom <x>"]), secret=prng.choice([None, "", "whsec_%06d_%s" % (i, "k" * prng.randrange(40))]))
            for i in range(N)]
    cb, co, dur, fl, rb, ro, sb, so = S.pack_webhook_deliveries(recs)
    cap = int(_abi.load().afc_webhook_bound(_abi.ptr(co), _abi.ptr(ro), N))
    out.append(("webhook", "afc_webhook_sign_batch", [In(cb), In(co), In(dur), In(fl), In(rb), In(ro), In(sb), In(so), N, Out(np.zeros(cap, np.uint8)), cap,
                                                      Out(np.zeros(N + 1, np.uint64)), Out(np.zeros((N, 71), np.uint8)), Out(np.zeros(N, np.uint8))],
                None, None))
    # DID registration
    dreqs = DC.random_requests(random.Random(11), N, max_ids=6)
    for i, r in enumerate(dreqs):
        r["agent_node_id"] = b"staged-node-%06d" % i
    nodes, node_off, id_idx, ids, id_off = DC.pack(dreqs)
    m = int(id_idx[-1])
    cap = int(_abi.load().afc_did_register_bound(_abi.ptr(node_off), _abi.ptr(id_idx), _abi.ptr(id_off), N, len(DC.SERVER)))
    args = [In(np.frombuffer(MASTER, np.uint8)), Host(DC.SERVER), len(DC.SERVER), In(nodes), In(node_off), In(np.arange(N, dtype=np.uint32)), In(id_idx),
            In(ids), In(id_off), N, Out(np.zeros(N + 1, np.uint64)), Out(np.zeros((N + m) * 96, np.uint8)), Out(np.zeros((N + m) * 32, np.uint8)),
            Out(np.zeros((N + m) * 55, np.uint8)), Out(np.zeros((N + m) * 48, np.uint8)), Out(np.zeros(N + m, np.uint8)), Out(np.zeros(cap, np.uint8)), cap,
            Out(np.zeros(N + 1, np.uint64))]
    out.append(("did_register", "afc_did_register_batch", args, None, None))
    return out, {"keysets": (ks, nks), "did_requests": dreqs}


def log_root(lib, log):
    root = (C.c_uint8 * 32)()
    size = C.c_uint64()
    assert lib.afc_merkle_root(log, root, C.byref(size)) == 0
    return bytes(root) + size.value.to_bytes(8, "little")


def main():
    """Every case in the three buffer modes and as its _dev call (run in a fresh process with 97-item chunks)."""
    import agentfield_b200 as afb
    from agentfield_b200 import _abi
    lib = _abi.load()
    ctx = afb.Context(0)

    def new_log():
        h = C.c_void_p()
        _abi.check(lib.afc_merkle_new(ctx.handle, C.byref(h)), ctx.handle)
        return h
    logs = {}

    def fresh(args, key):
        """The arguments with a new log in place of the marker (each run appends to its own log)."""
        return [logs.setdefault(key, new_log()) if a is LOG else a for a in args]
    LOG = C.c_void_p(1)
    cs, extra = cases(ctx, LOG)
    for name, fn, args, dfn, dargs in cs:
        runs = {mode: host_call(lib, ctx, fn, fresh(args, (name, mode)), mode) for mode in ("pageable", "pinned", "mixed")}
        runs["dev"] = dev_call(lib, ctx, dfn or fn + "_dev", fresh(dargs or args, (name, "dev")))
        if any(a is LOG for a in args):
            for mode in runs:
                runs[mode].append(np.frombuffer(log_root(lib, logs[(name, mode)]), np.uint8))
        for mode in ("pinned", "mixed", "dev"):
            assert len(runs[mode]) == len(runs["pageable"])
            for k, (a, b) in enumerate(zip(runs["pageable"], runs[mode])):
                assert a.tobytes() == b.tobytes(), (name, mode, k)
        print("ok", name, flush=True)
    for h in logs.values():
        lib.afc_merkle_free(h)
    for k in extra["keysets"]:
        k.close()
    print("staging modes ok")


def in_fresh_process(call, env=None):
    script = "import sys; sys.path[:0] = [sys.argv[1], sys.argv[1] + '/tests']; import test_host_staging_gpu as T; T.%s" % call
    r = subprocess.run([sys.executable, "-c", script, ROOT], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "ok\n" in r.stdout[-20:], r.stdout[-3000:] + r.stderr[-3000:]


def test_pinned_pageable_and_mixed_buffers_agree_with_dev_calls():
    """~1000 items in 97-item chunks (AFC_CHUNK_ITEMS is read once per process): each call wraps the slot ring more than twice."""
    in_fresh_process("main()", dict(os.environ, AFC_CHUNK_ITEMS="97", AFC_MIN_CHUNK_ITEMS="97"))


@pytest.mark.parametrize("mode", ["pageable", "pinned"])
def test_no_secret_left_in_staging(mode):
    """A fresh process, so that its context's staging memory holds only what these calls left."""
    in_fresh_process("no_secret_left(%r)" % mode)


def no_secret_left(mode):
    """After sign (seeds), webhook (secrets), pubkey / expand (seeds, expanded keys), sign-expanded, issue and workflow (expanded keys) and
    DID registration (master seed, derived keys, private JWKs), with the calls' buffers pageable or pinned, the staging memory of a fresh
    context holds none of those secrets; the public node ids DID registration staged are still found, which shows the search sees that
    memory."""
    import did_cases as DC
    import agentfield_b200 as afb
    from agentfield_b200 import _abi
    lib = _abi.load()
    ctx = afb.Context(0)
    cs, extra = cases(ctx, None)
    byname = {c[0]: c for c in cs}
    res = {name: host_call(lib, ctx, byname[name][1], byname[name][2], mode)
           for name in ("sign", "webhook", "pubkey", "expand", "sign_expanded", "sign_expanded_key_index", "issue", "workflow", "did_register")}

    def hits(pattern):
        h = C.c_uint64()
        _abi.check(lib.afc_staging_find(ctx.handle, pattern, len(pattern), C.byref(h)), ctx.handle)
        return h.value
    assert hits(b"staged-node-000123") > 0
    seeds, exp = byname["sign"][2][0].a, res["expand"][0].reshape(-1, 96)
    for i in range(0, N, 53):
        assert hits(seeds[i].tobytes()) == 0 and hits(exp[i, :32].tobytes()) == 0 and hits(exp[i, 32:64].tobytes()) == 0, i
    sb, so = byname["webhook"][2][6].a, byname["webhook"][2][7].a
    for i in range(N):
        secret = sb[int(so[i]):int(so[i + 1])].tobytes()
        assert len(secret) < 12 or hits(secret) == 0, secret
    derived = byname["issue"][2][0].a
    for k in range(derived.shape[0]):
        assert hits(derived[k, :32].tobytes()) == 0 and hits(derived[k, 32:64].tobytes()) == 0, k
    assert hits(MASTER) == 0
    comps = [c for w in DC.oracle(extra["did_requests"], 0, master=MASTER) for c in w["components"]]
    comp_off, expanded = res["did_register"][0].view(np.uint64), res["did_register"][1].reshape(-1, 96)
    assert int(comp_off[-1]) == len(comps)
    for c in range(0, len(comps), 97):
        assert hits(expanded[c, :32].tobytes()) == 0 and hits(expanded[c, 32:64].tobytes()) == 0, c
        assert hits(comps[c]["seed"]) == 0 and hits(base64.urlsafe_b64encode(comps[c]["seed"]).rstrip(b"=")) == 0, c
    for k in extra["keysets"]:
        k.close()
    print("no secret left ok")
