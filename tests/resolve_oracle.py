"""ORACLE for DID resolution and DID documents: DIDService.ResolveDID's scan (control-plane/internal/services/did_service.go:368-473) over a
Go-shaped registry and the c.JSON of both handlers (internal/handlers/did_handlers.go:73-94, 368-429) restated in Python, independent of
the package.  The root's JWK comes from oracle/ref_did.public_jwk; strings are escaped by oracle/go_json.escape_bytes and the document's
publicKeyJwk is json.Unmarshal into map[string]interface{} (Python's json module with Go's rules added) written back by
oracle/go_json.value_bytes.

A registry is {"root_did", "root_pk", "agents": [agent]}: an agent {"did", "derivation_path", "public_key_jwk", "reasoners", "skills"},
its two maps lists of (function name, component) pairs, a component {"did", "derivation_path", "public_key_jwk", "function_name"}; all
values bytes.  Go iterates the agents and both maps in random order, so for a DID held more than once every holder is a valid answer:
outcomes() returns them all."""
import json
import re

from oracle import go_json as OJ
from oracle import ref_did as RD

ROOT_PATH = b"m/44'/0'"
SERVER, AGENT, REASONER, SKILL = 0, 1, 2, 3
COMPONENT_TYPES = (b"agentfield_server", b"agent", b"reasoner", b"skill")
RESOLVE, DOCUMENT = 0, 1
CAP = 4096                     # a longer body is left to the host
JV_MAX_DEPTH = 32


def q(b: bytes) -> bytes:
    return b'"' + OJ.escape_bytes(b) + b'"'


def identities(reg):
    """Every identity ResolveDID can return, in scan order: the root, then each agent, its reasoners and its skills."""
    out = [{"did": reg["root_did"], "kind": SERVER, "derivation_path": ROOT_PATH, "function_name": b"", "public_key_jwk": RD.public_jwk(reg["root_pk"])}]
    for a in reg["agents"]:
        out.append({"did": a["did"], "kind": AGENT, "derivation_path": a["derivation_path"], "function_name": b"", "public_key_jwk": a["public_key_jwk"]})
        for kind, name in ((REASONER, "reasoners"), (SKILL, "skills")):
            for _, c in a[name]:
                out.append({"did": c["did"], "kind": kind, "derivation_path": c["derivation_path"], "function_name": c["function_name"],
                            "public_key_jwk": c["public_key_jwk"]})
    return out


def candidates(reg, did):
    """What ResolveDID(did) may return: the root alone when did is the root DID (it is checked first), else every holder of did."""
    ids = identities(reg)
    if did == reg["root_did"]:
        return [ids[0]]
    return [e for e in ids[1:] if e["did"] == did]


# ---- json.Unmarshal(raw, &map[string]interface{}) then json.Marshal

def _tokens_have_escaped_key(raw: bytes) -> bool:
    """A key written with a backslash (the device sorts keys by their input bytes, so it declines them)."""
    for m in re.finditer(rb'"((?:[^"\\]|\\.)*)"\s*:', raw, re.S):
        if b"\\" in m.group(1):
            return True
    return False


def _depth(raw: bytes) -> int:
    depth = best = 0
    in_str = esc = False
    for c in raw:
        if in_str:
            if esc:
                esc = False
            elif c == 0x5C:
                esc = True
            elif c == 0x22:
                in_str = False
        elif c == 0x22:
            in_str = True
        elif c in b"[{":
            depth += 1
            best = max(best, depth)
        elif c in b"]}":
            depth -= 1
    return best


def jwk_marshal(raw: bytes):
    """(ok, text, exact): ok False when json.Unmarshal into a map fails (a 500: the device leaves it to the host); else text is what
    json.Marshal writes back, and exact False marks the values the device may leave to the host instead (invalid UTF-8, lone surrogates,
    duplicate or escaped keys, nesting deeper than 32, numbers outside float64's normal range or with more than 19 digits).  text is None
    when Python cannot compute Go's text (invalid UTF-8)."""
    def no_const(x):
        raise ValueError(x)
    try:
        text = raw.decode("utf-8")
    except UnicodeDecodeError:
        return True, None, False
    flags = {"exact": True}

    def num(s):
        x = float(s)
        if x in (float("inf"), float("-inf")):
            raise ValueError("range")
        digits = re.sub(r"[eE].*", "", s).replace("-", "").replace(".", "").lstrip("0")
        if (x == 0 and digits) or (x != 0 and abs(x) < 2.2250738585072014e-308) or len(digits) > 19:
            flags["exact"] = False
        return x

    def pairs(p):
        keys = [k for k, _ in p]
        if len(set(keys)) != len(keys):
            flags["exact"] = False
        return dict(p)
    try:
        v = json.loads(text, parse_float=num, parse_int=num, parse_constant=no_const, object_pairs_hook=pairs)
    except ValueError:
        return False, None, True
    if v is not None and not isinstance(v, dict):
        return False, None, True

    def has_surrogate(x):
        if isinstance(x, str):
            return any(0xD800 <= ord(c) <= 0xDFFF for c in x)
        if isinstance(x, dict):
            return any(has_surrogate(k) or has_surrogate(y) for k, y in x.items())
        if isinstance(x, list):
            return any(has_surrogate(y) for y in x)
        return False
    if has_surrogate(v):
        return True, None, False
    exact = flags["exact"] and not _tokens_have_escaped_key(raw) and _depth(raw) <= JV_MAX_DEPTH
    return True, OJ.value_bytes(v), exact


# ---- the handlers' bodies

def resolve_body(e) -> bytes:
    return (b'{"component_type":"' + COMPONENT_TYPES[e["kind"]] + b'","derivation_path":' + q(e["derivation_path"]) + b',"did":' + q(e["did"]) +
            b',"function_name":' + q(e["function_name"]) + b',"public_key_jwk":' + q(e["public_key_jwk"]) + b"}")


def document_body(did: bytes, jwk_text: bytes) -> bytes:
    key = q(did + b"#key-1")
    return (b'{"@context":["https://www.w3.org/ns/did/v1","https://w3id.org/security/suites/ed25519-2020/v1"],"assertionMethod":[' + key +
            b'],"authentication":[' + key + b'],"id":' + q(did) + b',"service":[{"description":"AgentField Agent Platform Service","id":' +
            q(did + b"#agentfield-service") + b',"serviceEndpoint":"https://agentfield.example.com/api/v1","type":"AgentFieldAgentService"}],'
            b'"verificationMethod":[{"controller":' + q(did) + b',"id":' + key + b',"publicKeyJwk":' + jwk_text +
            b',"type":"Ed25519VerificationKey2020"}]}')


def outcome(kind, did, e):
    """(status, body, host_ok) of one request answered by identity e (None: not found).  body None: the device cannot write it (a 500,
    or text Python cannot compute); host_ok: the device may leave it to the host."""
    if not did:
        return 400, b'{"error":"DID parameter is required"}', False
    if e is None:
        if kind == RESOLVE:
            return 404, b'{"error":"DID not found"}', False
        return 404, b'{"details":' + q(b"DID not found: " + did) + b',"error":"DID not found"}', False
    if kind == RESOLVE:
        body = resolve_body(e)
        return 200, body, len(body) > CAP
    ok, text, exact = jwk_marshal(e["public_key_jwk"])
    if not ok:
        return 500, None, True
    if text is None:
        return 200, None, True
    body = document_body(did, text)
    return 200, body, not exact or len(body) > CAP


def outcomes(reg, kind, did):
    """Every (status, body, host_ok) the reference may give for the request."""
    cs = candidates(reg, did) if did else []
    if not cs:
        return [outcome(kind, did, None)]
    return [outcome(kind, did, e) for e in cs]


def accepts(outs, state, body) -> bool:
    """Whether a device answer (state AFC_DIDRES_*, body) is one of the outcomes: the exact body and status, or HOST where the host may
    (or, for a body over CAP, must) build it."""
    status = {0: 200, 1: 404, 2: 400}
    for st, b, host_ok in outs:
        if state == 3:
            if host_ok:
                return True
        elif b is not None and status.get(state) == st and body == b and (st != 200 or len(b) <= CAP):
            return True
    return False
