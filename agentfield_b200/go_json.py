"""Byte-exact restatement of Go `encoding/json.Marshal` for the structs that ARE the canonical signing form on the hot path
(control-plane/pkg/types/did_types.go:135-220, pkg/types/webhook.go:42-53).  Host-side string work: in the real
deployment this stays in Go (SURVEY.md §8a row V1); the Python mirror needs it so that the issue -> verify flow of
BASELINE.json configs[0] can be driven end to end through the GPU path with the same bytes Go would sign.

Rules restated (Go 1.24): struct fields in declaration order under their json tags; `omitempty` drops "" / nil;
strings escape `"` `\\` and control characters (\\b \\f \\n \\r \\t short forms, others \\u00XX), and — because Marshal
uses escapeHTML — `<` `>` `&` as \\u003c \\u003e \\u0026, plus U+2028 / U+2029; nil slices are `null`; map keys sorted;
float64 uses strconv's shortest digits in 'f' form, 'e' form (exponent without padding) when |x| < 1e-6 or >= 1e21; numbers that
went through json.Unmarshal into interface{} are float64 (unmarshal_numbers).
"""
import math
from decimal import Decimal

_ESC = {'"': '\\"', "\\": "\\\\", "\b": "\\b", "\f": "\\f", "\n": "\\n", "\r": "\\r", "\t": "\\t",
        "<": "\\u003c", ">": "\\u003e", "&": "\\u0026", "\u2028": "\\u2028", "\u2029": "\\u2029"}


def string(s: str) -> str:
    out = ['"']
    for ch in s:
        e = _ESC.get(ch)
        if e is not None:
            out.append(e)
        elif ch < " ":
            out.append("\\u%04x" % ord(ch))
        elif 0xD800 <= ord(ch) <= 0xDFFF:
            out.append("\\ufffd")            # invalid UTF-8 in Go becomes U+FFFD
        else:
            out.append(ch)
    out.append('"')
    return "".join(out)


def _shortest_digits(a: float):
    """(digits, point): a = d0.d1d2... x 10^point with `digits` the shortest decimal string that round-trips to the float64 a
    (what strconv.FormatFloat(a, fmt, -1, 64) starts from; Python's repr uses the same shortest-round-trip rule)."""
    _, digs, exp = Decimal(repr(float(a))).as_tuple()
    digs = list(digs)
    while len(digs) > 1 and digs[-1] == 0:
        digs.pop(); exp += 1
    while len(digs) > 1 and digs[0] == 0:
        digs.pop(0)
    return "".join(map(str, digs)), exp + len(digs) - 1


def number(x) -> str:
    """encoding/json floatEncoder (encode.go): strconv 'f' form with the shortest digits, 'e' form when |x| < 1e-6 or >= 1e21,
    the exponent cleaned up from e-09 to e-9.  Go ints (Python int) print as integers; bool is handled by value()."""
    if isinstance(x, bool):
        return "true" if x else "false"
    if isinstance(x, int):
        return str(x)
    if math.isnan(x) or math.isinf(x):
        raise ValueError("json: unsupported value: %r" % x)    # Go returns UnsupportedValueError
    if x == 0:
        return "-0" if math.copysign(1, x) < 0 else "0"
    sign = "-" if x < 0 else ""
    a = abs(x)
    d, pt = _shortest_digits(a)
    if a < 1e-6 or a >= 1e21:                                  # %e: d.ddde[+-]dd, then e-09 -> e-9
        mant = d[0] + ("." + d[1:] if len(d) > 1 else "")
        return "%s%se%s%s" % (sign, mant, "-" if pt < 0 else "+", str(abs(pt)) if abs(pt) >= 10 else "%d" % abs(pt))
    if pt >= len(d) - 1:                                       # %f, integer valued: digits then zeros, no point
        return sign + d + "0" * (pt - (len(d) - 1))
    if pt >= 0:
        return sign + d[:pt + 1] + "." + d[pt + 1:]
    return sign + "0." + "0" * (-pt - 1) + d


def unmarshal_interface(text):
    """json.Unmarshal(text, &interface{}): every number becomes a float64 — including "-0", which keeps its sign."""
    import json
    return json.loads(text, parse_int=float)


def unmarshal_numbers(v):
    """What json.Unmarshal into interface{} does to numbers: every one becomes a float64 (vc_service.go:250-251 parses the
    stored document before verifyVCSignature re-marshals it, so `metadata` values and webhook results round-trip through
    float64)."""
    if isinstance(v, bool) or v is None or isinstance(v, str):
        return v
    if isinstance(v, (int, float)):
        return float(v)
    if isinstance(v, dict):
        return {k: unmarshal_numbers(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [unmarshal_numbers(x) for x in v]
    raise TypeError("unsupported JSON value %r" % type(v))


def value(v) -> str:
    if v is None:
        return "null"
    if isinstance(v, str):
        return string(v)
    if isinstance(v, (bool, int, float)):
        return number(v)
    if isinstance(v, dict):
        return "{" + ",".join(string(k) + ":" + value(v[k]) for k in sorted(v)) + "}"
    if isinstance(v, (list, tuple)):
        return "[" + ",".join(value(x) for x in v) + "]"
    raise TypeError("unsupported JSON value %r" % type(v))


def string_list(xs) -> str:
    return "null" if xs is None else "[" + ",".join(string(x) for x in xs) + "]"


def vc_proof(p) -> str:
    return ('{"type":%s,"created":%s,"verificationMethod":%s,"proofPurpose":%s,"proofValue":%s}'
            % (string(p.get("type", "")), string(p.get("created", "")), string(p.get("verificationMethod", "")),
               string(p.get("proofPurpose", "")), string(p.get("proofValue", ""))))


EMPTY_PROOF = {"type": "", "created": "", "verificationMethod": "", "proofPurpose": "", "proofValue": ""}


def vc_document(doc, proof=None) -> bytes:
    """json.Marshal(types.VCDocument).  proof=None -> the zero-valued Proof the reference signs over (vc_service.go:436-439)."""
    cs = doc["credentialSubject"]
    ex = cs["execution"]
    execution = ('{"inputHash":%s,"outputHash":%s,"timestamp":%s,"durationMs":%d,"status":%s%s}'
                 % (string(ex["inputHash"]), string(ex["outputHash"]), string(ex["timestamp"]), int(ex["durationMs"]), string(ex["status"]),
                    (',"errorMessage":' + any_string(ex["errorMessage"])) if ex.get("errorMessage") else ""))
    au = cs["audit"]
    audit = '{"inputDataHash":%s,"outputDataHash":%s,"metadata":%s}' % (string(au["inputDataHash"]), string(au["outputDataHash"]), value(au.get("metadata")))
    ca, ta = cs["caller"], cs["target"]
    subject = ('{"executionId":%s,"workflowId":%s,"sessionId":%s,"caller":{"did":%s,"type":%s,"agentNodeDid":%s},'
               '"target":{"did":%s,"agentNodeDid":%s,"functionName":%s},"execution":%s,"audit":%s}'
               % (string(cs["executionId"]), string(cs["workflowId"]), string(cs["sessionId"]), string(ca["did"]), string(ca["type"]),
                  string(ca["agentNodeDid"]), string(ta["did"]), string(ta["agentNodeDid"]), string(ta["functionName"]), execution, audit))
    return ('{"@context":%s,"type":%s,"id":%s,"issuer":%s,"issuanceDate":%s,"credentialSubject":%s,"proof":%s}'
            % (string_list(doc["@context"]), string_list(doc["type"]), string(doc["id"]), string(doc["issuer"]), string(doc["issuanceDate"]),
               subject, vc_proof(proof if proof is not None else EMPTY_PROOF))).encode("utf-8")


def truncate_error_message(msg):
    """vc_service.go:153-160: `if len(msg) > 500 { msg = msg[:500] + "...[truncated]" }` — len and the slice count BYTES.  A cut
    inside a UTF-8 sequence leaves invalid bytes that json.Marshal then writes as \ufffd, one per byte.  Returns what Go's string
    would hold, as bytes (str in -> bytes out only when truncated); string_bytes() renders it."""
    if msg is None:
        return None
    raw = msg.encode("utf-8", "surrogatepass") if isinstance(msg, str) else bytes(msg)
    if len(raw) <= 500:
        return msg
    return raw[:500] + b"...[truncated]"


def string_bytes(raw: bytes) -> str:
    """json.Marshal of a Go string holding arbitrary bytes: valid UTF-8 as string(), every byte of an invalid sequence as \ufffd
    (encode.go appendString + utf8.DecodeRune)."""
    out, i = ['"'], 0
    while i < len(raw):
        b = raw[i]
        if b < 0x80:
            out.append(string(chr(b))[1:-1]); i += 1
            continue
        n = 2 if 0xC2 <= b <= 0xDF else 3 if 0xE0 <= b <= 0xEF else 4 if 0xF0 <= b <= 0xF4 else 0
        try:
            if n == 0:
                raise UnicodeDecodeError("utf-8", raw, i, i + 1, "lead")
            out.append(string(raw[i:i + n].decode("utf-8"))[1:-1]); i += n       # strict: overlongs, surrogates, > U+10FFFF raise
        except UnicodeDecodeError:
            out.append("\\ufffd"); i += 1
    out.append('"')
    return "".join(out)


def any_string(s) -> str:
    return string_bytes(bytes(s)) if isinstance(s, (bytes, bytearray)) else string(s)


def workflow_vc_document(doc, proof=None) -> bytes:
    """json.Marshal(types.WorkflowVCDocument) (pkg/types/did_types.go:146-180; built by createWorkflowVCDocument,
    vc_service.go:635-683; marshalled with a zero Proof by signWorkflowVC :686-693 and verifyWorkflowVCSignature :1589-1597,
    with the proof for storage :611).  componentVcIds is a []string (nil -> null), totalSteps / completedSteps are ints,
    endTime is *string with omitempty (absent when nil, present — even as "" — otherwise)."""
    cs = doc["credentialSubject"]
    orc, au = cs["orchestrator"], cs["audit"]
    end = ',"endTime":' + string(cs["endTime"]) if cs.get("endTime") is not None else ""
    subject = ('{"workflowId":%s,"sessionId":%s,"componentVcIds":%s,"totalSteps":%d,"completedSteps":%d,"status":%s,"startTime":%s%s,'
               '"snapshotTime":%s,"orchestrator":{"did":%s,"type":%s,"agentNodeDid":%s},'
               '"audit":{"inputDataHash":%s,"outputDataHash":%s,"metadata":%s}}'
               % (string(cs["workflowId"]), string(cs["sessionId"]), string_list(cs["componentVcIds"]), int(cs["totalSteps"]),
                  int(cs["completedSteps"]), string(cs["status"]), string(cs["startTime"]), end, string(cs["snapshotTime"]),
                  string(orc["did"]), string(orc["type"]), string(orc["agentNodeDid"]),
                  string(au["inputDataHash"]), string(au["outputDataHash"]), value(au.get("metadata"))))
    return ('{"@context":%s,"type":%s,"id":%s,"issuer":%s,"issuanceDate":%s,"credentialSubject":%s,"proof":%s}'
            % (string_list(doc["@context"]), string_list(doc["type"]), string(doc["id"]), string(doc["issuer"]), string(doc["issuanceDate"]),
               subject, vc_proof(proof if proof is not None else EMPTY_PROOF))).encode("utf-8")


def webhook_payload(p) -> bytes:
    """json.Marshal(types.ExecutionWebhookPayload) (pkg/types/webhook.go:42-53)."""
    parts = ['"event":' + string(p["event"]), '"execution_id":' + string(p["execution_id"]), '"workflow_id":' + string(p["workflow_id"]),
             '"status":' + string(p["status"]), '"target":' + string(p["target"]), '"type":' + string(p["type"])]
    if p.get("duration_ms") is not None:
        parts.append('"duration_ms":%d' % int(p["duration_ms"]))
    if p.get("result") is not None:
        parts.append('"result":' + value(p["result"]))
    if p.get("error_message") is not None:
        parts.append('"error_message":' + string(p["error_message"]))
    parts.append('"timestamp":' + string(p["timestamp"]))
    return ("{" + ",".join(parts) + "}").encode("utf-8")


def go_utf8(raw: bytes) -> str:
    """A Go string's bytes as Python text the way Go's decoder reads them: valid UTF-8 as itself, every byte utf8.DecodeRune rejects as
    U+FFFD, one per byte."""
    out, i = [], 0
    while i < len(raw):
        b = raw[i]
        if b < 0x80:
            out.append(chr(b)); i += 1
            continue
        n = 2 if 0xC2 <= b <= 0xDF else 3 if 0xE0 <= b <= 0xEF else 4 if 0xF0 <= b <= 0xF4 else 0
        try:
            if n == 0:
                raise UnicodeDecodeError("utf-8", raw, i, i + 1, "lead")
            out.append(raw[i:i + n].decode("utf-8")); i += n
        except UnicodeDecodeError:
            out.append("�"); i += 1
    return "".join(out)


def _no_surrogates(v):
    """Lone surrogate escapes decode to U+FFFD in Go; a key that becomes equal to another one then overwrites it (last wins)."""
    if isinstance(v, str):
        return "".join("�" if 0xD800 <= ord(c) <= 0xDFFF else c for c in v)
    if isinstance(v, dict):
        out = {}
        for k, x in v.items():
            out[_no_surrogates(k)] = _no_surrogates(x)
        return out
    if isinstance(v, list):
        return [_no_surrogates(x) for x in v]
    return v


def _go_float(text):
    x = float(text)
    if math.isinf(x):
        raise ValueError("json: cannot unmarshal number %s into a float64" % text)    # strconv.ParseFloat range error
    return x


def _reject_constant(name):
    raise ValueError("invalid character in JSON: %s" % name)                            # NaN / Infinity are not JSON


def decode_execution_payload(raw):
    """decodeExecutionPayload (internal/services/webhook_dispatcher.go:459-468) with Go's rules, not Python's: None for empty raw (nil);
    the decoded interface{} value (numbers float64, None for null) when json.Unmarshal accepts raw; otherwise the bytes of raw (the
    Go string(raw)).  Unmarshal rejects invalid syntax (NaN and Infinity included) and numbers out of float64 range."""
    import json
    raw = bytes(raw or b"")
    if not raw:
        return None
    try:
        v = json.loads(go_utf8(raw), parse_float=_go_float, parse_int=_go_float, parse_constant=_reject_constant)
    except ValueError:
        return raw
    return _no_surrogates(v)


def webhook_event(status) -> str:
    """determineWebhookEvent (webhook_dispatcher.go:450-457)."""
    from .services import normalize_execution_status
    s = go_utf8(status) if isinstance(status, (bytes, bytearray)) else status
    return "execution.completed" if normalize_execution_status(s) == "succeeded" else "execution.failed"


def build_webhook_payload(record) -> bytes:
    """json.Marshal(buildPayload(exec, determineWebhookEvent(exec.Status))) (webhook_dispatcher.go:296-299, 394-419).  record: execution_id,
    run_id, status, node_id, reasoner_id, target_type, timestamp (str or bytes); duration_ms (int or None); result (the raw stored
    ResultPayload, bytes; None or b"" = nil); error_message (str, bytes or None)."""
    def col(k):
        v = record[k]
        return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)
    event = webhook_event(record["status"])
    parts = ['"event":' + string(event), '"execution_id":' + string_bytes(col("execution_id")), '"workflow_id":' + string_bytes(col("run_id")),
             '"status":' + string_bytes(col("status")), '"target":' + string_bytes(col("node_id") + b"." + col("reasoner_id")),
             '"type":' + string_bytes(col("target_type"))]
    if record.get("duration_ms") is not None:
        parts.append('"duration_ms":%d' % int(record["duration_ms"]))
    if event == "execution.completed":
        r = decode_execution_payload(record.get("result"))
        if isinstance(r, bytes):
            parts.append('"result":' + string_bytes(r))
        elif r is not None:
            parts.append('"result":' + value(r))
    elif record.get("error_message") is not None:
        parts.append('"error_message":' + string_bytes(col("error_message")))
    parts.append('"timestamp":' + string_bytes(col("timestamp")))
    return ("{" + ",".join(parts) + "}").encode("utf-8")
