"""ORACLE for VC verification requests: POST /api/v1/did/verify (control-plane/internal/handlers/did_handlers.go:97-111) with gin v1.10.1's
default binding and VCService.VerifyVC (internal/services/vc_service.go:242-289), restated in Python from the reference and from the
documented behaviour of Go 1.24's encoding/json and encoding/base64, independent of the package and of the device:

  bind      json.NewDecoder(body).Decode(&types.VCVerificationRequest): Go's scanner reads the first value whole (a syntax error anywhere in
            it is a 400, bytes after it are never read, depth is limited to 10 000); a value other than an object or null does not decode
            into the struct (a 400); the struct field vc_document takes the last member whose unquoted name is "vc_document" or equal to
            it under foldName; json.RawMessage keeps the value's bytes
  verify    json.Unmarshal of those bytes into types.VCDocument (pkg/types/did_types.go:135-220), ResolveDID against a {did: public key}
            registry, json.Marshal with the zero proof (oracle/ref_vc.go_marshal), base64.RawURLEncoding of proofValue, ed25519.Verify
            (oracle/go_ed25519)
  response  c.JSON: {"error":"Invalid request body"} or json.Marshal(types.VCVerificationResponse) (did_types.go:273-279, omitempty), strings
            escaped by oracle/go_json.escape_bytes

answer(body, registry) returns (state, body bytes) with state OK (200) or BAD_REQUEST (400), or None where the oracle does not pin Go's
text: a document json.Unmarshal rejects for a type mismatch inside it (UnmarshalTypeError's field path is not restated here)."""
import base64
import functools
import json

from oracle import go_ed25519 as GE
from oracle import go_json as OJ
from oracle import ref_vc as RV

OK, BAD_REQUEST, HOST = 0, 1, 2
MAX_DEPTH = 10000
BAD_BODY = b'{"error":"Invalid request body"}'
_WS = b" \t\n\r"


class _SyntaxError(Exception):
    pass


def _string_end(b, i):
    """b[i] is an opening quote: the index after the closing one (Go's scanner: no byte below 0x20, the nine escapes)."""
    i += 1
    while True:
        if i >= len(b):
            raise _SyntaxError("unexpected end")
        c = b[i]
        if c == 0x22:
            return i + 1
        if c < 0x20:
            raise _SyntaxError("control character in string")
        if c == 0x5C:
            if i + 1 >= len(b):
                raise _SyntaxError("unexpected end")
            e = b[i + 1]
            if e == ord("u"):
                h = b[i + 2:i + 6]
                if len(h) < 4:
                    raise _SyntaxError("unexpected end")
                if any(x not in b"0123456789abcdefABCDEF" for x in h):
                    raise _SyntaxError("bad \\u escape")
                i += 6
                continue
            if e not in b'"\\/bfnrt':
                raise _SyntaxError("bad escape")
            i += 2
            continue
        i += 1


def _number_end(b, i):
    j = i
    if j < len(b) and b[j] == 0x2D:
        j += 1
    digits = lambda k: k < len(b) and 0x30 <= b[k] <= 0x39    # noqa: E731
    if not digits(j):
        raise _SyntaxError("bad number")
    if b[j] == 0x30:
        j += 1
    else:
        while digits(j):
            j += 1
    if j < len(b) and b[j] == 0x2E:
        j += 1
        if not digits(j):
            raise _SyntaxError("bad fraction")
        while digits(j):
            j += 1
    if j < len(b) and b[j] in b"eE":
        j += 1
        if j < len(b) and b[j] in b"+-":
            j += 1
        if not digits(j):
            raise _SyntaxError("bad exponent")
        while digits(j):
            j += 1
    return j


def first_value(b):
    """(start, end) of the first JSON value of b as Go's Decoder reads it, or raises _SyntaxError (io.EOF included)."""
    i = 0
    while i < len(b) and b[i] in _WS:
        i += 1
    if i == len(b):
        raise _SyntaxError("EOF")
    start = i
    stack = []                     # "{" / "[" of the open containers
    expect_value = True
    while True:
        while i < len(b) and b[i] in _WS:
            i += 1
        if i >= len(b):
            if not stack and not expect_value:
                return start, i
            raise _SyntaxError("unexpected end")
        c = b[i]
        if expect_value:
            if c in b"{[":
                if len(stack) >= MAX_DEPTH:
                    raise _SyntaxError("exceeded max depth")
                stack.append(c)
                i += 1
                while i < len(b) and b[i] in _WS:
                    i += 1
                if i < len(b) and b[i] == (0x7D if c == 0x7B else 0x5D):
                    stack.pop()
                    i += 1
                    expect_value = False
                    if not stack:
                        return start, i
                    continue
                if c == 0x7B:
                    i = _member_name(b, i)
                continue
            if c == 0x22:
                i = _string_end(b, i)
            elif c in b"-0123456789":
                i = _number_end(b, i)
            else:
                for w in (b"true", b"false", b"null"):
                    if c == w[0]:
                        if b[i:i + len(w)] != w:
                            raise _SyntaxError("bad literal")
                        i += len(w)
                        break
                else:
                    raise _SyntaxError("invalid character")
            expect_value = False
            if not stack:
                return start, i
            continue
        top = stack[-1]
        if c == 0x2C:
            i += 1
            if top == 0x7B:
                i = _member_name(b, i)
            expect_value = True
            continue
        if c == (0x7D if top == 0x7B else 0x5D):
            stack.pop()
            i += 1
            if not stack:
                return start, i
            continue
        raise _SyntaxError("after value")


def _member_name(b, i):
    """Whitespace, a quoted name, whitespace and a colon from i; the index after the colon."""
    while i < len(b) and b[i] in _WS:
        i += 1
    if i >= len(b) or b[i] != 0x22:
        raise _SyntaxError("expected name")
    i = _string_end(b, i)
    while i < len(b) and b[i] in _WS:
        i += 1
    if i >= len(b) or b[i] != 0x3A:
        raise _SyntaxError("expected colon")
    return i + 1


def fold_name(name: str) -> str:
    """encoding/json foldName (Go 1.24): ASCII letters upper-cased, any other rune r mapped to unicode.ToUpper(unicode.ToLower(r))."""
    out = []
    for ch in name:
        if ch < "\x80":
            out.append(ch.upper() if "a" <= ch <= "z" else ch)
            continue
        lo = ch.lower() if len(ch.lower()) == 1 else ch
        up = lo.upper() if len(lo.upper()) == 1 else lo
        out.append(up)
    return "".join(out)


class _NegZero(int):
    """The integer token -0: 0 as a Go int, -0 as a float64."""


def _go_text(raw: bytes) -> str:
    """The bytes as Go's decoder sees them: each byte of invalid UTF-8 stands for U+FFFD."""
    out, i = [], 0
    while i < len(raw):
        size, ok = OJ._decode_rune(raw, i) if raw[i] >= 0x80 else (1, True)
        out.append(raw[i:i + size].decode("utf-8") if ok else "\ufffd")
        i += size if ok else 1
    return "".join(out)


def _no_surrogates(v):
    """json.Unmarshal writes a lone surrogate escape as U+FFFD."""
    if isinstance(v, str):
        return "".join("\ufffd" if 0xD800 <= ord(c) <= 0xDFFF else c for c in v)
    if isinstance(v, list):
        return [_no_surrogates(x) for x in v]
    if isinstance(v, tuple):
        return ("obj", [(_no_surrogates(k), _no_surrogates(x)) for k, x in v[1]])
    return v


def _decode(raw: bytes):
    return _no_surrogates(json.loads(_go_text(raw), object_pairs_hook=lambda kv: ("obj", kv),
                                     parse_int=lambda t: _NegZero(0) if t == "-0" else int(t)))


def bind(body: bytes):
    """("bad",) for a bind error; ("absent",) without a vc_document (or for a top-level null); ("value", raw bytes of the winning member)."""
    try:
        a, e = first_value(body)
    except _SyntaxError:
        return ("bad",)
    text = body[a:e]
    if text[:1] == b"n":
        return ("absent",)
    if text[:1] != b"{":
        return ("bad",)
    # the members of the top-level object, with each value's raw bytes: walk the object with first_value on each value
    found = ("absent",)
    i = 1
    while True:
        while text[i] in _WS:
            i += 1
        if text[i] == 0x7D:
            return found
        if text[i] == 0x2C:
            i += 1
            while text[i] in _WS:
                i += 1
        k1 = _string_end(text, i)
        name = _no_surrogates(json.loads(_go_text(text[i:k1])))
        i = _member_name(text, i)
        v0, v1 = first_value(text[i:])
        if name == "vc_document" or fold_name(name) == fold_name("vc_document"):
            found = ("value", text[i + v0:i + v1])
        i += v1


# ---- VerifyVC
_S, _L, _I, _M = "string", "[]string", "int", "map"
_VCDOC = [("@context", _L), ("type", _L), ("id", _S), ("issuer", _S), ("issuanceDate", _S),
          ("credentialSubject", [("executionId", _S), ("workflowId", _S), ("sessionId", _S),
                                 ("caller", [("did", _S), ("type", _S), ("agentNodeDid", _S)]),
                                 ("target", [("did", _S), ("agentNodeDid", _S), ("functionName", _S)]),
                                 ("execution", [("inputHash", _S), ("outputHash", _S), ("timestamp", _S), ("durationMs", _I), ("status", _S),
                                                ("errorMessage", _S)]),
                                 ("audit", [("inputDataHash", _S), ("outputDataHash", _S), ("metadata", _M)])]),
          ("proof", [("type", _S), ("created", _S), ("verificationMethod", _S), ("proofPurpose", _S), ("proofValue", _S)])]


class _TypeMismatch(Exception):
    pass


def _zero(t):
    if isinstance(t, list):
        return {k: _zero(x) for k, x in t}
    return {_S: "", _I: 0}.get(t)


def _iface(v):
    if isinstance(v, tuple) and v[:1] == ("obj",):
        return {k: _iface(x) for k, x in v[1]}
    if isinstance(v, list):
        return [_iface(x) for x in v]
    if isinstance(v, _NegZero):
        return -0.0
    if isinstance(v, int) and not isinstance(v, bool):
        return float(v)
    return v


def _into(v, t, cur):
    """json.Unmarshal of the decoded value v into a Go value of type t holding cur."""
    is_obj = isinstance(v, tuple) and v[:1] == ("obj",)
    if isinstance(t, list):
        if v is None:
            return cur
        if not is_obj:
            raise _TypeMismatch()
        names = [k for k, _ in t]
        for k, x in v[1]:
            f = k if k in names else next((n for n in names if fold_name(n) == fold_name(k)), None)
            if f is not None:
                cur[f] = _into(x, dict(t)[f], cur[f])
        return cur
    if v is None:
        return None if t in (_L, _M) else cur
    if t == _S:
        if not isinstance(v, str):
            raise _TypeMismatch()
        return v
    if t == _L:
        if not isinstance(v, list) or not all(x is None or isinstance(x, str) for x in v):
            raise _TypeMismatch()
        return ["" if x is None else x for x in v]
    if t == _I:
        if isinstance(v, bool) or not isinstance(v, int) or not -2**63 <= v < 2**63:
            raise _TypeMismatch()
        return int(v)
    if not is_obj:
        raise _TypeMismatch()
    return _iface(v)


def _marshal_zero_proof(d):
    ex = dict(d["credentialSubject"]["execution"])
    if not ex["errorMessage"]:
        del ex["errorMessage"]
    cs = dict(d["credentialSubject"], execution=ex)
    cs["audit"] = dict(cs["audit"], metadata=RV.sorted_map(cs["audit"]["metadata"]))
    doc = dict(d, credentialSubject=cs, proof=_zero(_VCDOC[-1][1]))
    return RV.go_marshal(doc)


def b64_error_at(s: bytes):
    """base64.RawURLEncoding.DecodeString(s): None if it decodes, else the CorruptInputError offset: the first byte outside the URL alphabet
    (\\r and \\n skipped), else, for a count of alphabet bytes = 1 mod 4, the last byte of s."""
    alpha = b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789-_"
    count = 0
    for k, c in enumerate(s):
        if c in b"\r\n":
            continue
        if c not in alpha:
            return k
        count += 1
    return len(s) - 1 if count % 4 == 1 else None


@functools.lru_cache(maxsize=1 << 16)
def _verify(pk, msg, sig):
    """ed25519.Verify.  OpenSSL (through `cryptography`) answers first, as it is fast; its only disagreements with Go are signatures with
    small-order or non-canonical points, so a signature it accepts is confirmed by oracle/go_ed25519 and one it rejects stands."""
    if len(sig) != 64:
        return False
    from cryptography.exceptions import InvalidSignature
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PublicKey
    try:
        Ed25519PublicKey.from_public_bytes(pk).verify(sig, msg)
    except (InvalidSignature, ValueError):
        return GE.verify(pk, msg, sig) if _small_order_r(sig) else False
    return GE.verify(pk, msg, sig)


def _small_order_r(sig):
    return sig[:32] in GE.small_order_points()


def verify_vc(raw: bytes, registry):
    """VCService.VerifyVC(raw) as a VCVerificationResponse dict (missing keys = omitted), or None where the oracle does not pin the text."""
    if raw is None:
        return {"valid": False, "error": "failed to parse VC document: unexpected end of JSON input"}
    v = _decode(raw)
    if isinstance(v, (str, bool, list, int, float)):
        what = "string" if isinstance(v, str) else "bool" if isinstance(v, bool) else "array" if isinstance(v, list) else "number"
        return {"valid": False, "error": "failed to parse VC document: json: cannot unmarshal %s into Go value of type types.VCDocument" % what}
    try:
        d = _into(v, _VCDOC, _zero(_VCDOC))
    except _TypeMismatch:
        return None
    iss = d["issuer"]
    if iss not in registry:
        return {"valid": False, "error": "failed to resolve issuer DID: DID not found: " + iss}
    pv = d["proof"]["proofValue"].encode("utf-8")
    k = b64_error_at(pv)
    if k is not None:
        return {"valid": False, "error": "failed to verify signature: failed to decode signature: illegal base64 data at input byte %d" % k}
    sig = base64.urlsafe_b64decode(pv.replace(b"\r", b"").replace(b"\n", b"") + b"=" * (-len(pv.replace(b"\r", b"").replace(b"\n", b"")) % 4))
    if not _verify(registry[iss], _marshal_zero_proof(d), sig):
        return {"valid": False, "message": "Invalid signature"}
    return {"valid": True, "issuer_did": iss, "issued_at": d["issuanceDate"], "message": "VC verified successfully"}


def response_bytes(r) -> bytes:
    out = b'{"valid":' + (b"true" if r["valid"] else b"false")
    for k in ("issuer_did", "issued_at", "message", "error"):
        if r.get(k):
            out += b',"' + k.encode() + b'":"' + OJ.escape_bytes(r[k].encode("utf-8")) + b'"'
    return out + b"}"


def answer(body: bytes, registry):
    """(state, response bytes) for one request body, or None (see the module docstring).  registry: {did str: 32-byte public key}."""
    b = bind(body)
    if b[0] == "bad":
        return BAD_REQUEST, BAD_BODY
    r = verify_vc(b[1] if b[0] == "value" else None, registry)
    return None if r is None else (OK, response_bytes(r))
