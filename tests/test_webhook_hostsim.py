"""The webhook routines (agentfield_b200/csrc/afc_float.cuh, afc_jsonval.cuh, afc_webhook.cuh), compiled for the CPU
(tests/hostsim/hostsim_webhook.cpp), against Python's correctly rounded float parsing, the host mirror (agentfield_b200/go_json.py) and the
golden deliveries: float64 parsing and formatting, json.Marshal(json.Unmarshal(raw)) in every spelling, the named declines, texts
Unmarshal rejects, whole bodies and headers, and the event rule."""
import ctypes as C
import json
import math
import os
import random
import re
import struct
import subprocess

import numpy as np
import pytest

from conftest import golden
from agentfield_b200 import go_json as GJ, services as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = -1


@pytest.fixture(scope="module")
def wh(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("whsim") / "libafc_whsim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_webhook.cpp")])
    lib = C.CDLL(out)
    lib.hs_fl_parse.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p]
    lib.hs_fl_format.argtypes = [C.c_uint64, C.c_void_p]
    lib.hs_fl_format.restype = C.c_uint32
    lib.hs_fl_parse_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.hs_fl_format_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    lib.hs_jv_validate.argtypes = [C.c_char_p, C.c_uint64]
    lib.hs_jv_validate.restype = C.c_uint32
    lib.hs_jv_emit.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p, C.c_uint64]
    lib.hs_jv_emit.restype = C.c_int64
    lib.hs_wh_delivery.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_uint32, C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint32, C.c_void_p,
                                   C.c_uint64, C.c_void_p]
    lib.hs_wh_delivery.restype = C.c_int64
    lib.hs_wh_fixed_bytes.restype = C.c_uint64
    return lib


def bits_of(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def parse(wh, text):
    b = C.c_uint64()
    return b.value if wh.hs_fl_parse(text, len(text), C.byref(b)) else None


def fmt(wh, x):
    out = (C.c_uint8 * 64)()
    n = wh.hs_fl_format(bits_of(x), out)
    return bytes(out)[:n].decode()


def spellings(x):
    r = repr(x)
    e = "%.17e" % x
    mant, ex = e.split("e")
    out = [r, "%.17g" % x, "%.20e" % x, e.replace("e", "E"), mant + "e+" + ex.lstrip("+") if not ex.startswith("-") else e,
           mant + "e" + ex[0] + "00" + ex[1:], mant.rstrip("0") + "000e" + ex]
    return [s.replace("inf", "x") for s in out]


def expected_host(x):
    """Inputs the device may leave to the host: subnormal and zero results of non-zero text, overflow."""
    a = abs(x)
    return a == 0 or a < 2.2250738585072014e-308 or math.isinf(a)


def test_parse_random_bit_patterns(wh):
    rng = np.random.default_rng(0x3E8)
    bits = rng.integers(0, 2 ** 64, 10 ** 6, dtype=np.uint64)
    xs = bits.view(np.float64)
    xs = xs[np.isfinite(xs)]
    texts, expect = [], []
    for x in xs.tolist():
        for t in spellings(x):
            texts.append(t.encode())
            expect.append(float(t))
    buf = np.frombuffer(b"".join(texts), dtype=np.uint8)
    off = np.zeros(len(texts) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(t) for t in texts])
    ok = np.zeros(len(texts), dtype=np.uint8)
    got = np.zeros(len(texts), dtype=np.uint64)
    wh.hs_fl_parse_batch(buf.ctypes.data, off.ctypes.data, len(texts), ok.ctypes.data, got.ctypes.data)
    exp = np.array(expect, dtype=np.float64).view(np.uint64)
    assert (got[ok == 1] == exp[ok == 1]).all()
    declined = [expect[i] for i in np.nonzero(ok == 0)[0]]
    give_ups = [x for x in declined if not expected_host(x)]
    assert len(give_ups) <= 10, give_ups[:10]            # Eisel-Lemire give-ups for this seed, per million bit patterns


@pytest.mark.parametrize("text", ["0.5", "1.5", "2.5", "0.1", "9007199254740991", "9007199254740992", "9007199254740993", "9007199254740994",
                                  "9007199254740995", "1e23", "8.98846567431158e307", "1.7976931348623157e308", "2.2250738585072014e-308",
                                  "1234567890123456789", "12345678901234567890", "123456789012345678901234567890", "1.00000000000000011102230246251565404",
                                  "0.30000000000000004", "-0", "-0.0", "0e-999", "4.35", "1e-6", "9.999999999999999e20", "1e21",
                                  "0.000000000000000000000000000000000001", "100000000000000000000000000000000000000000000"])
def test_parse_hand_picked(wh, text):
    b = parse(wh, text.encode())
    if b is None:        # a give-up is allowed only at (or, past 19 digits, within the truncation of) a halfway point between two float64s
        assert text in ("9007199254740993", "9007199254740995", "1.00000000000000011102230246251565404")
        return
    assert b == bits_of(float(text)), text


@pytest.mark.parametrize("text", ["1e400", "-1e400", "1e309", "1e-400", "5e-324", "2.225073858507201e-308", "1.7976931348623159e308"])
def test_parse_declines_out_of_normal_range(wh, text):
    assert parse(wh, text.encode()) is None


def test_format_random_and_boundaries(wh):
    rng = np.random.default_rng(0x3E9)
    bits = rng.integers(0, 2 ** 64, 200000, dtype=np.uint64)
    xs = [x for x in bits.view(np.float64).tolist() if math.isfinite(x) and (x == 0 or abs(x) >= 2.2250738585072014e-308)]
    xs += [1e-6, 9.999999e-7, math.nextafter(1e-6, 0), math.nextafter(1e-6, 1), 1e21, math.nextafter(1e21, 0), 1e20, 0.0, -0.0, 1.7976931348623157e308,
           2.2250738585072014e-308, 2.0 ** 53, 123456789.125, 5e-7, 1.5e-10]
    xs += [float("%de%d" % (d, e)) for d in (1, 3, 7, 9) for e in range(-307, 308)]
    xs += [m * 10.0 ** e for m in (1.2345678901234567, 9.876543210987654) for e in range(-300, 300, 7)]
    arr = np.array(xs, dtype=np.float64).view(np.uint64)
    out = np.zeros(len(xs) * 32, dtype=np.uint8)
    ln = np.zeros(len(xs), dtype=np.uint8)
    wh.hs_fl_format_batch(arr.ctypes.data, len(xs), out.ctypes.data, ln.ctypes.data)
    for i, x in enumerate(xs):
        assert bytes(out[32 * i:32 * i + int(ln[i])]).decode() == GJ.number(x), x
    for f in golden("go_cases.json")["floats"]:
        x = struct.unpack(">d", bytes.fromhex(f["bits"]))[0]
        if x == 0 or abs(x) >= 2.2250738585072014e-308:
            assert fmt(wh, x) == f["expect"]


def emit(wh, raw):
    out = (C.c_uint8 * (6 * len(raw) + 64))()
    n = wh.hs_jv_emit(raw, len(raw), out, len(out))
    assert n != -2 and n != -3
    return HOST if n == -1 else bytes(out)[:n]


def random_value(rng, depth=0):
    k = rng.random()
    if depth < 5 and k < 0.15:
        return {rng.choice(["a", "b", "key", "Zeta", "é", "中文", "x<y", "k_%d" % rng.randrange(50), ""]) + str(rng.randrange(3)): random_value(rng, depth + 1)
                for _ in range(rng.randrange(6))}
    if depth < 5 and k < 0.25:
        return [random_value(rng, depth + 1) for _ in range(rng.randrange(6))]
    if k < 0.45:
        return "".join(rng.choice(["a", " ", "<", ">", "&", '"', "\\", "\n", "\x01", "é", "😀", " ", "/", "\x7f"]) for _ in range(rng.randrange(12)))
    if k < 0.65:
        return rng.choice([rng.uniform(-1e6, 1e6), rng.random() * 10.0 ** rng.randrange(-30, 30), float(rng.randrange(-10 ** 6, 10 ** 6))])
    if k < 0.8:
        return rng.randrange(-10 ** 20, 10 ** 20)
    return rng.choice([None, True, False])


def test_values_in_every_spelling(wh):
    rng = random.Random(0x3EA)
    seen = 0
    for _ in range(3000):
        v = random_value(rng)
        for sp in (dict(), dict(separators=(",", ":")), dict(indent=2), dict(ensure_ascii=False), dict(indent="\t", ensure_ascii=False)):
            raw = json.dumps(v, **sp).encode("utf-8")
            got = emit(wh, raw)
            want = GJ.value(GJ.decode_execution_payload(raw)).encode("utf-8")
            if got == HOST:      # only escaped keys (ensure_ascii spellings of non-ASCII keys) and give-ups past 19 digits
                assert b'\\' in raw or re.search(rb"\d{20}", raw), raw
                continue
            seen += 1
            assert got == want, raw
    assert seen > 6000


@pytest.mark.parametrize("raw", [b'{"a":1,"a":2}', b'{"b":{"x":1,"x":1}}', b'{"k\\u00e9y":1}', b'{"a\\"b":1}', b'"\\ud800"', b'"\\udc00 x"',
                                 b'"\\ud800\\u0041"', b'"\xff"', b'{"\xc3":1}', b'["a\xe4\xb8"]', b"[" * 33 + b"]" * 33, b"1e400", b"-1e309",
                                 b"1e-400", b"[5e-324]", b'{"x":2.2250738585072e-310}'])
def test_named_declines(wh, raw):
    assert wh.hs_jv_validate(raw, len(raw)) in (0, 2)
    assert wh.hs_jv_validate(raw, len(raw)) == 2 or emit(wh, raw) == HOST


def test_depth_32_is_built(wh):
    raw = b"[" * 32 + b"1" + b"]" * 32
    assert emit(wh, raw) == raw


@pytest.mark.parametrize("raw", [b'{"a":1,}', b"NaN", b"Infinity", b"{'a': 1}", b"01", b"1.", b".5", b"-", b"+1", b'"a\x01b"', b"\xef\xbb\xbf{}",
                                 b"   ", b"1 2", b"[1,]", b"tru", b"nul", b'{"a" 1}', b'{"a":}', b"[", b'"abc', b'"\\x"', b'"\\u12g4"', b"\x0b1",
                                 b"1e", b"1e+", b"-01", b"[1]]"])
def test_invalid_json_is_carried_as_a_string(wh, raw):
    assert wh.hs_jv_validate(raw, len(raw)) == 1
    assert isinstance(GJ.decode_execution_payload(raw), bytes)


def wh_delivery(wh, rec):
    cb, co, dur, fl, rb, ro, sb, so = S.pack_webhook_deliveries([rec])
    res = bytes(rec.get("result") or b"")
    sec = bytes(sb[:int(so[1])]) if rec.get("secret") is not None else b""
    cap = 6 * (len(cb) + len(res)) + int(wh.hs_wh_fixed_bytes()) + 64
    out, hd = (C.c_uint8 * cap)(), (C.c_uint8 * 71)()
    n = wh.hs_wh_delivery(cb.ctypes.data, co.ctypes.data, int(dur[0]), int(fl[0]), res, len(res), sec, len(sec), out, cap, hd)
    if n == HOST:
        return HOST
    return {"body": bytes(out)[:n], "header": bytes(hd).decode() if rec.get("secret") is not None else None}


def golden_records():
    """go_cases.json["webhooks"] (the payload struct, event rule applied: a failed event carries no result) and webhook_cases.json."""
    out = []
    for c in golden("go_cases.json")["webhooks"]:
        if c["event"] == "execution.failed" and c["result_json"] is not None:
            continue                                     # buildPayload never sets Result on a failed event
        node, fn = c["target"].rsplit(".", 1)
        out.append(dict(execution_id=c["execution_id"], run_id=c["workflow_id"], status=c["status"], node_id=node, reasoner_id=fn, target_type=c["type"],
                        timestamp=c["timestamp"], duration_ms=c["duration_ms"], error_message=c["error_message"], secret=c["secret"],
                        result=None if c["result_json"] is None else c["result_json"].encode(), expect_body=c["expect_body"],
                        expect_header=c["expect_header"]))
    for c in golden("webhook_cases.json"):
        out.append(dict(c, result=c["result"].encode("utf-8")))
    return out


def test_golden_bodies_and_headers(wh):
    built = 0
    for rec in golden_records():
        want = {"body": rec["expect_body"].encode("utf-8"), "header": rec["expect_header"]}
        assert S.sign_webhook_delivery_host(rec) == want
        got = wh_delivery(wh, rec)
        if got != HOST:
            built += 1
            assert got == want, rec["execution_id"]
    assert built >= 80


STATUSES = ["unknown", "pending", "queued", "running", "succeeded", "failed", "cancelled", "timeout", "success", "successful", "completed", "complete",
            "done", "ok", "error", "failure", "errored", "canceled", "cancel", "timed_out", "wait", "waiting", "in_progress", "processing"]


def test_event_rule(wh):
    base = dict(execution_id="e", run_id="r", node_id="n", reasoner_id="f", target_type="reasoner", timestamp="t", duration_ms=None,
                error_message="x", result=b"1", secret=None)
    for s in STATUSES:
        for v in (s, s.upper(), s.title(), " %s\t" % s, "\n%s\r" % s.upper(), "\x0b%s\x0c" % s, s + "x", ""):
            rec = dict(base, status=v)
            got = wh_delivery(wh, rec)
            assert got != HOST
            assert got["body"] == GJ.build_webhook_payload(rec), v
            assert (b'"event":"execution.completed"' in got["body"]) == (S.normalize_execution_status(v) == "succeeded")
    for v in ("succeeded\x85", "ok\xa0", "Kok", "done\x1c"):
        assert wh_delivery(wh, dict(base, status=v)) == HOST


def test_fixed_text_bounds_the_body(wh):
    rec = dict(execution_id="", run_id="", status="ok", node_id="", reasoner_id="", target_type="", timestamp="", duration_ms=-2 ** 63,
               error_message="", result=b'""', secret=None)
    assert len(wh_delivery(wh, rec)["body"]) <= wh.hs_wh_fixed_bytes()
    rec = dict(rec, status="failed")
    assert len(wh_delivery(wh, rec)["body"]) <= wh.hs_wh_fixed_bytes()
