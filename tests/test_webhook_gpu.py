"""afc_webhook_sign_batch[_dev] on the GPU against the host mirror (agentfield_b200/go_json.py build_webhook_payload), the CPU build of
the same routines (tests/hostsim/hostsim_webhook.cpp) and hmac: golden deliveries, random batches in every result spelling, host-buffer
versus device calls (also with 97-delivery chunks), argument errors, empty and all-declined batches, and 2^20 deliveries."""
import hashlib
import hmac
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from agentfield_b200 import _abi, go_json as GJ, services as S

pytestmark = pytest.mark.gpu

from test_webhook_hostsim import golden_records, random_value, wh, wh_delivery  # noqa: E402,F401  (the CPU build fixture)

RESULTS = [b'{"answer": "42 <ok>", "score": 0.8700000000000001, "items": [1, 2.5, null, true], "nested": {"z": 1e21, "a": 1e-7}}',
           b'{"b":2,"a":1}', b'[1e20, -0.0, 12345678901234567890]', b'"just a string"', b"12.5", b"null", b"false", b'""', b"0",
           b"NaN", b"{'a': 1}", b"   ", b"1 2", b'{"a":1,}', b"\xef\xbb\xbf{}", b'{"a":1,"a":2}', b'"\\ud800"', b"1e400", b"[" * 40 + b"]" * 40,
           b"", b"\xff\xfe", b'{"k\\u00e9y": 1}']
STATUSES = ["succeeded", "failed", " Success ", "DONE", "error", "ok", "completed", "timeout", "running", "done\x85"]


def random_records(n, seed):
    rng = random.Random(seed)
    recs = []
    for i in range(n):
        if rng.random() < 0.5:
            v = random_value(rng)
            sp = rng.choice([dict(), dict(separators=(",", ":")), dict(indent=2), dict(ensure_ascii=False)])
            res = json.dumps(v, **sp).encode()
        else:
            res = rng.choice(RESULTS)
        recs.append(dict(execution_id="exec_%d" % i, run_id=rng.choice(["run_1", "run_<2>", "r ", "r\xe9"]), status=rng.choice(STATUSES),
                         node_id=rng.choice(["node", "n\xff".encode("latin-1"), "節"]), reasoner_id="fn_%d" % (i % 7),
                         target_type=rng.choice(["reasoner", "skill"]), timestamp="2026-09-21T06:30:%02dZ" % (i % 60),
                         duration_ms=rng.choice([None, 0, rng.randrange(-2 ** 63, 2 ** 63)]), result=res,
                         error_message=rng.choice([None, "", "boom <x> & \"y\"", "é" * 300]),
                         secret=rng.choice([None, "", "whsec_%d" % i, "k" * rng.randrange(1, 200)])))
    return recs


def as_results(bodies, off, headers, status, recs):
    out = []
    for i, r in enumerate(recs):
        if status[i] == _abi.WEBHOOK_HOST:
            assert off[i + 1] == off[i] and not headers[i].any()
            out.append(None)
        else:
            out.append({"body": bytes(bodies[int(off[i]):int(off[i + 1])]),
                        "header": headers[i].tobytes().decode() if r.get("secret") is not None else None})
            if r.get("secret") is None:
                assert not headers[i].any()
    return out


def dev_call(ctx, packed, cap=None):
    import torch
    cb, co, dur, fl, rb, ro, sb, so = packed
    n = len(ro) - 1
    dev = torch.device("cuda", ctx.device)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    bound = int(ctx._lib.afc_webhook_bound(_abi.ptr(co), _abi.ptr(ro), n))
    d_bodies = torch.empty(max(bound, 1), dtype=torch.uint8, device=dev)
    d_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    d_h = torch.empty((n, 71), dtype=torch.uint8, device=dev)
    d_st = torch.empty(n, dtype=torch.uint8, device=dev)
    ins = [t(cb), t(co.view(np.int64)), t(dur), t(fl), t(rb), t(ro.view(np.int64)), t(sb), t(so.view(np.int32))]
    ctx.webhook_sign_dev(*ins, n, d_bodies, bound if cap is None else cap, d_off, d_h, d_st)
    torch.cuda.synchronize(dev)
    off = d_off.cpu().numpy().view(np.uint64)
    return d_bodies.cpu().numpy()[:int(off[-1]) if n else 0], off, d_h.cpu().numpy(), d_st.cpu().numpy()


def test_golden(ctx):
    recs = golden_records()
    got = S.sign_webhook_deliveries_batch(recs, ctx)
    assert got == [{"body": r["expect_body"].encode("utf-8"), "header": r["expect_header"]} for r in recs]
    bodies, off, headers, status = ctx.webhook_sign_packed(*S.pack_webhook_deliveries(recs))
    assert (status == _abi.WEBHOOK_BUILT).sum() >= 80


def test_random_deliveries_equal_mirror_and_cpu_build(ctx, wh):
    recs = random_records(20000, 0x3EB)
    res = as_results(*ctx.webhook_sign_packed(*S.pack_webhook_deliveries(recs)), recs)
    host = 0
    for r, g in zip(recs, res):
        cpu = wh_delivery(wh, r)
        if g is None:
            host += 1
            assert cpu == -1
            continue
        assert g == cpu == S.sign_webhook_delivery_host(r), r
    assert 0 < host < len(recs) // 2


def test_host_and_device_calls_agree(ctx):
    recs = random_records(3000, 0x3EC)
    packed = S.pack_webhook_deliveries(recs)
    a = ctx.webhook_sign_packed(*packed)
    b = dev_call(ctx, packed)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_chunk_boundaries_in_a_fresh_process():
    """The host-buffer call with chunks of 97 deliveries (AFC_CHUNK_ITEMS is read once per process)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, AFC_CHUNK_ITEMS="97", AFC_MIN_CHUNK_ITEMS="97")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(root, "tests", "test_webhook_gpu.py"), "-m", "gpu", "-q", "-x", "-p", "no:cacheprovider",
                        "-k", "golden or host_and_device"], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def test_argument_errors(ctx):
    recs = random_records(5, 0x3ED)
    cb, co, dur, fl, rb, ro, sb, so = S.pack_webhook_deliveries(recs)
    n = 5
    lib = ctx._lib
    bound = int(lib.afc_webhook_bound(_abi.ptr(co), _abi.ptr(ro), n))
    bodies = np.full(bound + 16, 0xA5, dtype=np.uint8)
    boff = np.zeros(n + 1, dtype=np.uint64)
    hd = np.zeros((n, 71), dtype=np.uint8)
    st = np.full(n, 9, dtype=np.uint8)

    def call(cap, co=co, ro=ro, so=so, fl=fl, nn=n, b=bodies):
        return lib.afc_webhook_sign_batch(ctx.handle, _abi.ptr(cb), _abi.ptr(co), _abi.ptr(dur), _abi.ptr(fl), _abi.ptr(rb), _abi.ptr(ro), _abi.ptr(sb),
                                          _abi.ptr(so), nn, _abi.ptr(b), cap, _abi.ptr(boff), _abi.ptr(hd), _abi.ptr(st))
    assert call(bound - 1) == _abi.AFC_EINVAL
    assert (bodies == 0xA5).all() and (st == 9).all()              # nothing written
    back = co.copy(); back[3] = back[2] - 1 if back[2] else 0; back[2] += 1
    assert call(bound, co=back) == _abi.AFC_EINVAL
    rback = ro.copy(); rback[2], rback[3] = rback[3], rback[2]
    if rback[2] != rback[3]:
        assert call(bound, ro=rback) == _abi.AFC_EINVAL
    sback = so.copy(); sback[1] = sback[2] + 1
    assert call(bound, so=sback) == _abi.AFC_EINVAL
    assert call(bound, fl=(fl | 0x80).astype(np.uint8)) == _abi.AFC_EINVAL
    assert (st == 9).all()
    assert lib.afc_webhook_sign_batch(None, _abi.ptr(cb), _abi.ptr(co), _abi.ptr(dur), _abi.ptr(fl), _abi.ptr(rb), _abi.ptr(ro), _abi.ptr(sb),
                                      _abi.ptr(so), n, _abi.ptr(bodies), bound, _abi.ptr(boff), _abi.ptr(hd), _abi.ptr(st)) == _abi.AFC_EINVAL
    assert call(bound) == _abi.AFC_OK
    with pytest.raises(_abi.AfcError):
        dev_call(ctx, (cb, co, dur, fl, rb, ro, sb, so), cap=bound - 1)


def test_empty_and_all_host_batches(ctx):
    assert S.sign_webhook_deliveries_batch([], ctx) == []
    bodies, off, headers, status = ctx.webhook_sign_packed(*S.pack_webhook_deliveries([]))
    assert len(off) == 1 and off[0] == 0 and len(status) == 0
    recs = [dict(r, status="done\x85") for r in random_records(300, 0x3EE)]
    bodies, off, headers, status = ctx.webhook_sign_packed(*S.pack_webhook_deliveries(recs))
    assert (status == _abi.WEBHOOK_HOST).all() and off[-1] == 0 and not headers.any()
    assert S.sign_webhook_deliveries_batch(recs, ctx) == [S.sign_webhook_delivery_host(r) for r in recs]


def test_one_million_deliveries(ctx):
    base = random_records(4096, 0x3EF)
    n = 1 << 20
    recs = [base[i % 4096] for i in range(n)]
    cb, co, dur, fl, rb, ro, sb, so = S.pack_webhook_deliveries(recs)
    bodies, off, headers, status = dev_call(ctx, (cb, co, dur, fl, rb, ro, sb, so))
    assert int(off[-1]) == len(bodies)
    secrets = [None if r.get("secret") is None else S._wh_bytes(r["secret"]) for r in base]
    for i in range(n):
        if status[i] == _abi.WEBHOOK_BUILT and secrets[i % 4096] is not None:
            body = bodies[int(off[i]):int(off[i + 1])].tobytes()
            assert headers[i].tobytes() == b"sha256=" + hmac.new(secrets[i % 4096], body, hashlib.sha256).hexdigest().encode()
    rng = random.Random(5)
    for i in rng.sample(range(n), 2000):
        r = recs[i]
        if status[i] == _abi.WEBHOOK_HOST:
            assert status[i % 4096] == _abi.WEBHOOK_HOST
            continue
        assert bodies[int(off[i]):int(off[i + 1])].tobytes() == GJ.build_webhook_payload(r)
