"""ORACLE for workflow VC chains: GetWorkflowVCChain (control-plane/internal/services/vc_service.go:292-338) with
collectDIDResolutionBundle (:810-870) and the handler's c.JSON (internal/handlers/ui/did.go:383) restated in Python, independent of the
package.  The workflow credential comes from oracle/ref_vc.py (through workflow_cases.oracle_docs); strings are escaped by
oracle/go_json.escape_bytes; vc_document goes through a restatement of Go's appendCompact(dst, src, escapeHTML=true) after a checkValid
built on Python's json module; times through datetime for Time.MarshalJSON.

A case is a workflow_cases case ({"cols": 7 byte strings, "records": [...]}) whose records are dicts: vc_id, status, sec, nsec, zone
(created_at's UTC offset in seconds), cols (13 byte strings in AFC_CHAIN_RECORD_COLUMNS order), flags (AFC_CHAIN_*_NIL bits), doc_size;
plus wf_vc_id, resolved_at (bytes) and clock (seconds, nanoseconds, UTC offset: the snapshot time)."""
import datetime as dt
import json

import workflow_cases as WC
from oracle import go_json as OJ

REC_COLUMNS = ("execution_id", "workflow_id", "session_id", "agent_node_id", "workflow_name", "issuer_did", "target_did", "caller_did",
               "vc_document", "signature", "storage_uri", "input_hash", "output_hash")
AGENT_NIL, NAME_NIL, DOC_NIL = 1, 2, 4
RESOLVED_MAX = 64
DID_MAX = 128
# unicode.IsSpace
SPACES = set("\t\n\v\f\r \x85\xa0\u1680\u2028\u2029\u202f\u205f\u3000") | {chr(c) for c in range(0x2000, 0x200B)}


def issue_case(case):
    """The case as afc_vc_issue_workflow_batch sees it."""
    return {"cols": case["cols"], "records": [(r["vc_id"], r["status"], r["sec"], r["nsec"]) for r in case["records"]]}


def s(b: bytes) -> bytes:
    return b'"' + OJ.escape_bytes(b) + b'"'


def time_ok(sec, nsec, zone):
    if not 0 <= nsec < 10 ** 9 or zone % 60 or not -86400 < zone < 86400:
        return False
    return WC.SEC_MIN <= sec + zone <= WC.SEC_MAX


def marshal_time(sec, nsec, zone) -> bytes:
    """Time.MarshalJSON: RFC3339Nano in the time's own zone."""
    t = dt.datetime(1970, 1, 1, tzinfo=dt.timezone.utc) + dt.timedelta(seconds=sec)
    t = t.astimezone(dt.timezone(dt.timedelta(seconds=zone)))
    out = "%04d-%02d-%02dT%02d:%02d:%02d" % (t.year, t.month, t.day, t.hour, t.minute, t.second)
    if nsec:
        out += ("." + "%09d" % nsec).rstrip("0")
    if zone == 0:
        out += "Z"
    else:
        a = abs(zone) // 60
        out += "%s%02d:%02d" % ("-" if zone < 0 else "+", a // 60, a % 60)
    return out.encode()


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


def check_valid(raw: bytes) -> bool:
    """Go's checkValid (RFC 8259; invalid UTF-8 inside strings is accepted), and no deeper than the device parses (32)."""
    def no_const(x):
        raise ValueError(x)
    try:
        json.loads(raw.decode("utf-8", "surrogateescape"), parse_constant=no_const)
    except ValueError:
        return False
    return _depth(raw) <= 32


def append_compact(raw: bytes) -> bytes:
    """appendCompact(dst, src, escapeHTML=true) of a valid text."""
    out = bytearray()
    in_str = esc = False
    i = 0
    while i < len(raw):
        c = raw[i]
        if c in b"<>&":
            out += b"\\u00" + b"%02x" % c
        elif c == 0xE2 and i + 2 < len(raw) and raw[i + 1] == 0x80 and raw[i + 2] in (0xA8, 0xA9):
            out += b"\\u202" + (b"8" if raw[i + 2] == 0xA8 else b"9")
            i += 3
            continue
        elif in_str:
            out.append(c)
            if esc:
                esc = False
            elif c == 0x5C:
                esc = True
            elif c == 0x22:
                in_str = False
        elif c in b" \t\n\r":
            pass
        else:
            out.append(c)
            in_str = c == 0x22
        i += 1
    return bytes(out)


def record_json(r) -> bytes:
    c = dict(zip(REC_COLUMNS, r["cols"]))
    parts = [b'"vc_id":' + s(r["vc_id"]), b'"execution_id":' + s(c["execution_id"]), b'"workflow_id":' + s(c["workflow_id"]),
             b'"session_id":' + s(c["session_id"])]
    if not r["flags"] & AGENT_NIL:
        parts.append(b'"agent_node_id":' + s(c["agent_node_id"]))
    if not r["flags"] & NAME_NIL:
        parts.append(b'"workflow_name":' + s(c["workflow_name"]))
    parts += [b'"issuer_did":' + s(c["issuer_did"]), b'"target_did":' + s(c["target_did"]), b'"caller_did":' + s(c["caller_did"]),
              b'"vc_document":' + (b"null" if r["flags"] & DOC_NIL else append_compact(c["vc_document"])),
              b'"signature":' + s(c["signature"]), b'"storage_uri":' + s(c["storage_uri"]), b'"document_size_bytes":%d' % r["doc_size"],
              b'"input_hash":' + s(c["input_hash"]), b'"output_hash":' + s(c["output_hash"]), b'"status":' + s(r["status"]),
              b'"created_at":"' + marshal_time(r["sec"], r["nsec"], r["zone"]) + b'"']
    return b"{" + b",".join(parts) + b"}"


def is_space_only(d: bytes) -> bool:
    text = d.decode("utf-8", "replace")
    return all(ch in SPACES for ch in text)


def method(d: bytes) -> bytes:
    return d.split(b":")[1] if len(d) > 4 and d[:4] == b"did:" else b"key"


def jwk_x(pk: bytes) -> bytes:
    import base64
    return base64.urlsafe_b64encode(pk).rstrip(b"=")


def bundle(case, directory) -> dict:
    """collectDIDResolutionBundle: DID -> public key for the DIDs the directory ({did: pk}) resolves."""
    col = REC_COLUMNS.index
    dids = [r["cols"][col(k)] for r in case["records"] for k in ("issuer_did", "caller_did", "target_did")] + [case["cols"][2]]
    out = {}
    for d in dids:
        if d in (b"", b"did:key:") or is_space_only(d) or d not in directory:
            continue
        out[d] = directory[d]
    return out


def is_host(case, directory):
    if WC.is_host(issue_case(case)) or not time_ok(*case["clock"]) or len(case["resolved_at"]) > RESOLVED_MAX:
        return True
    for r in case["records"]:
        if not time_ok(r["sec"], r["nsec"], r["zone"]):
            return True
        if not r["flags"] & DOC_NIL and not check_valid(r["cols"][REC_COLUMNS.index("vc_document")]):
            return True
    return any(len(d) > DID_MAX for d in bundle(case, directory))


def chain_body(case, directory, doc=None, proof_value=WC.PLACEHOLDER):
    """json.Marshal(WorkflowVCChainResponse) of a built workflow; doc: the stored workflow credential (default: the oracle's with
    proof_value)."""
    ic = issue_case(case)
    summ = WC.summary(ic)
    if doc is None:
        doc = WC.oracle_docs(ic, proof_value)[1]
    recs = case["records"]
    status = [k for k, v in WC.STATUS_IDS.items() if v == summ[0]][0].encode()
    cols = case["cols"]
    start = (recs[summ[2]]["sec"], recs[summ[2]]["nsec"], recs[summ[2]]["zone"]) if recs else case["clock"]
    wf = [b'"workflow_id":' + s(cols[0]), b'"session_id":' + s(cols[1]), b'"component_vcs":[' + b",".join(s(r["vc_id"]) for r in recs) + b"]",
          b'"workflow_vc_id":' + s(case["wf_vc_id"]), b'"status":' + s(status), b'"start_time":"' + marshal_time(*start) + b'"']
    if summ[3] != WC.NONE:
        e = recs[summ[3]]
        wf.append(b'"end_time":"' + marshal_time(e["sec"], e["nsec"], e["zone"]) + b'"')
    wf += [b'"total_steps":%d' % len(recs), b'"completed_steps":%d' % summ[1], b'"vc_document":' + doc, b'"signature":' + s(proof_value.encode())]
    if cols[2]:
        wf.append(b'"issuer_did":' + s(cols[2]))
    wf += [b'"snapshot_time":"' + marshal_time(*case["clock"]) + b'"', b'"storage_uri":""', b'"document_size_bytes":%d' % len(doc)]
    top = [b'"workflow_id":' + s(cols[0]), b'"component_vcs":[' + b",".join(record_json(r) for r in recs) + b"]",
           b'"workflow_vc":{' + b",".join(wf) + b"}", b'"total_steps":%d' % len(recs), b'"status":' + s(status)]
    b = bundle(case, directory)
    if b:
        ents = []
        for d in sorted(b):                                       # Go sorts map keys by their bytes before escaping them
            ents.append(s(d) + b':{"method":' + s(method(d)) + b',"public_key_jwk":{"alg":"EdDSA","crv":"Ed25519","kty":"OKP","use":"sig","x":"' +
                        jwk_x(b[d]) + b'"},"resolved_from":"bundled","resolved_at":' + s(case["resolved_at"]) + b"}")
        top.append(b'"did_resolution_bundle":{' + b",".join(ents) + b"}")
    return b"{" + b",".join(top) + b"}"
