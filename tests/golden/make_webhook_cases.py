"""Writes tests/golden/webhook_cases.json: whole webhook deliveries pinned through the oracle's construction (oracle/ref_vc.py).
Run by hand (python tests/golden/make_webhook_cases.py); the other fixtures come from make_golden.py and are not touched here."""
import json
import os
import sys

OUT = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(OUT))
sys.path.insert(0, ROOT)

from oracle import go_hash as H  # noqa: E402


def dump(name, obj):
    with open(os.path.join(OUT, name), "w") as f:
        json.dump(obj, f, indent=1, sort_keys=True)
        f.write("\n")


# ----------------------------------------------------------------------------- webhook deliveries built on the device
def make_webhook_cases():
    """webhook_cases.json: whole deliveries as buildPayload + json.Marshal + generateWebhookSignature produce them
    (internal/services/webhook_dispatcher.go:294-320, 394-474), every expectation through the oracle's construction
    (oracle/ref_vc.py webhook_payload / unmarshal_interface / go_marshal).  Results in the spellings agents send (Python json.dumps:
    default, compact, indent=2, ensure_ascii on and off, shuffled keys), floats from go_cases.json, top-level scalars, null / false / "",
    texts json.Unmarshal rejects (carried as a string), both events, nil and zero durations, with and without a secret."""
    import random
    from oracle import ref_vc as RV
    rng = random.Random(0xAF0E)
    floats = [struct_unpack_hex(f["bits"]) for f in json.load(open(os.path.join(OUT, "go_cases.json")))["floats"]]
    values = [{"answer": "42 <ok> & done", "score": 0.87, "n": 3, "items": [1e21, 1e-7, 2.5, None, True, False], "nested": {"z": 1, "a": {"k\u00e9y": "é中😀"}}},
              {"floats": floats[:30]}, {"floats": floats[30:]}, [{"b": 1, "a": 2}, [], {}, "\u2028\u2029", 12345678901234567890],
              "just a string", 12.5, 0, -0.0, 1e20, None, False, "", True, [], {}]
    spellings = [dict(), dict(separators=(",", ":")), dict(indent=2), dict(ensure_ascii=False), dict(indent=2, ensure_ascii=False)]
    texts = []
    for v in values:
        for sp in spellings:
            if isinstance(v, dict) and v:
                ks = list(v)
                rng.shuffle(ks)
                v = {k: v[k] for k in ks}
            texts.append(json.dumps(v, **sp))
    texts += ["", "NaN", "{'a': 1}", '{"a":1,}', "01", "1.", ".5", "-", "+1", "[1 2]", "\ufeff{}", "   ", "1 2", '"raw \x01 control"', "{\"a\":tru}"]
    statuses = ["succeeded", "failed", " Success ", "DONE", "error", "ok", "completed", "timeout"]
    out = []
    for i, t in enumerate(texts):
        st = statuses[i % len(statuses)]
        completed = RV_normalize(st) == "succeeded"
        try:
            res = RV.unmarshal_interface(t) if t else None
            if isinstance(res, float) and res != res:
                raise ValueError
            kind = "value"
        except ValueError:
            res, kind = t, "string"
        p_ = {"event": "execution.completed" if completed else "execution.failed", "execution_id": "exec_%d" % i, "workflow_id": "run_<%d>" % (i // 3),
              "status": st, "target": "node-%d.reasoner_%d" % (i % 4, i % 5), "type": "skill" if i % 3 == 0 else "reasoner",
              "duration_ms": None if i % 7 == 0 else (0 if i % 7 == 1 else 1000 * i - 7),
              "result": (res if kind == "value" else t) if completed and t else None,
              "error_message": None if completed or i % 4 == 0 else ("" if i % 4 == 1 else "boom <%d> & \"q\"" % i),
              "timestamp": "2026-09-21T06:%02d:%02dZ" % (i // 60, i % 60)}
        body = RV.go_marshal(RV.webhook_payload(p_))
        secret = None if i % 5 == 2 else "whsec_%d_" % i + "s" * (i % 90)
        out.append({"execution_id": p_["execution_id"], "run_id": p_["workflow_id"], "status": st, "node_id": "node-%d" % (i % 4),
                    "reasoner_id": "reasoner_%d" % (i % 5), "target_type": p_["type"], "timestamp": p_["timestamp"], "duration_ms": p_["duration_ms"],
                    "result": t, "error_message": p_["error_message"], "secret": secret, "expect_body": body.decode("utf-8"),
                    "expect_header": None if secret is None else H.webhook_signature(secret, body)})
    dump("webhook_cases.json", out)


def struct_unpack_hex(h):
    import struct
    return struct.unpack(">d", bytes.fromhex(h))[0]


def RV_normalize(status):
    aliases = {"success": "succeeded", "successful": "succeeded", "completed": "succeeded", "complete": "succeeded", "done": "succeeded", "ok": "succeeded"}
    s = status.strip().lower()
    return aliases.get(s, s)


if __name__ == "__main__":
    make_webhook_cases()
    print("webhook_cases.json written to", OUT)
