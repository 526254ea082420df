"""Canonical form on the device (SURVEY.md §8f N3): the bytes the reference signs and stores are json.Marshal of fixed
structs (VCDocument, control-plane/pkg/types/did_types.go:135-220, marshalled at internal/services/vc_service.go:436-439 for
signing and :201 for storage), i.e. constant text interleaved with a fixed number of values.  `JsonTemplate` holds the constant
text on the GPU and `fill_dev` assembles n documents from n x F values with Go's string escaping (afc_json_fill_*_dev), so a
batch can go  field values -> canonical bytes -> SHA-512 / Ed25519  without the documents ever existing on the host.

`vc_document_template()` is that struct's template; `vc_document_values()` lists one document's values in template order, so
`JsonTemplate.fill([...])` equals `go_json.vc_document(doc[, proof])` byte for byte (tests/test_gpu_parity.py)."""
import ctypes as C

import numpy as np

from . import _abi, go_json
from .crypto import default_context

STRING, RAW = 0, 1


class JsonTemplate:
    def __init__(self, segments, kinds, ctx=None):
        import torch
        if len(segments) != len(kinds) + 1:
            raise ValueError("a template of F values has F + 1 constant segments")
        self.ctx = ctx or default_context()
        self._lib = _abi.load()
        self.n_fields = len(kinds)
        self.segments, self.kinds = [bytes(s) for s in segments], list(kinds)
        dev = torch.device("cuda", self.ctx.device)
        seg = np.frombuffer(b"".join(self.segments) + b"\0", dtype=np.uint8).copy()
        off = np.zeros(len(segments) + 1, dtype=np.uint32)
        off[1:] = np.cumsum([len(s) for s in self.segments])
        self.d_segs = torch.from_numpy(seg).to(dev)
        self.d_seg_off = torch.from_numpy(off.view(np.int32)).to(dev)
        self.d_kinds = torch.tensor(list(kinds) or [0], dtype=torch.uint8, device=dev)

    def fill_dev(self, d_fields, d_field_off, n, stream=None):
        """d_fields: uint8 tensor of all values back to back; d_field_off: int64 tensor, n*F+1 offsets.  Returns (d_out uint8
        tensor, d_out_off int64 tensor of n+1 offsets), both on the device."""
        import torch
        dev = d_field_off.device
        d_out_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        total = C.c_uint64()
        st = self.ctx._stream(stream)
        _abi.check(self._lib.afc_json_fill_sizes_dev(self.ctx.handle, _abi.ptr(self.d_segs), _abi.ptr(self.d_seg_off), _abi.ptr(self.d_kinds),
                                                     self.n_fields, _abi.ptr(d_fields), _abi.ptr(d_field_off), n, _abi.ptr(d_out_off),
                                                     C.byref(total), st), self.ctx.handle)
        d_out = torch.empty(max(total.value, 1), dtype=torch.uint8, device=dev)
        _abi.check(self._lib.afc_json_fill_dev(self.ctx.handle, _abi.ptr(self.d_segs), _abi.ptr(self.d_seg_off), _abi.ptr(self.d_kinds),
                                               self.n_fields, _abi.ptr(d_fields), _abi.ptr(d_field_off), n, _abi.ptr(d_out_off), _abi.ptr(d_out),
                                               st), self.ctx.handle)
        return d_out[:total.value], d_out_off

    def pack_values(self, items):
        """items: n lists of F byte strings -> (fields uint8 array, offsets uint64 array of n*F+1)."""
        flat = [v for it in items for v in it]
        if len(flat) != len(items) * self.n_fields:
            raise ValueError("every item needs exactly %d values" % self.n_fields)
        off = np.zeros(len(flat) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(v) for v in flat], dtype=np.uint64)
        return np.frombuffer(b"".join(flat) + b"\0", dtype=np.uint8).copy(), off

    def fill(self, items):
        """Host convenience: n lists of F byte strings -> n documents (bytes), assembled on the GPU."""
        import torch
        n = len(items)
        if n == 0:
            return []
        dev = torch.device("cuda", self.ctx.device)
        fields, off = self.pack_values(items)
        d_out, d_off = self.fill_dev(torch.from_numpy(fields).to(dev), torch.from_numpy(off.view(np.int64)).to(dev), n)
        torch.cuda.synchronize(dev)
        out, o = d_out.cpu().numpy().tobytes(), d_off.cpu().numpy()
        return [out[int(o[i]):int(o[i + 1])] for i in range(n)]


def vc_document_template(with_proof=False, ctx=None):
    """Template of json.Marshal(types.VCDocument) on the GPU (see vc_document_template_parts)."""
    return JsonTemplate(*vc_document_template_parts(with_proof), ctx)


def vc_document_template_parts(with_proof=False):
    """(segments, kinds) of json.Marshal(types.VCDocument).  Without proof values the zero-valued Proof object the reference
    signs over (vc_service.go:436-439) is part of the constant text."""
    S, R = STRING, RAW
    parts = [('{"@context":', R), (',"type":', R), (',"id":"', S), ('","issuer":"', S), ('","issuanceDate":"', S),
             ('","credentialSubject":{"executionId":"', S), ('","workflowId":"', S), ('","sessionId":"', S),
             ('","caller":{"did":"', S), ('","type":"', S), ('","agentNodeDid":"', S),
             ('"},"target":{"did":"', S), ('","agentNodeDid":"', S), ('","functionName":"', S),
             ('"},"execution":{"inputHash":"', S), ('","outputHash":"', S), ('","timestamp":"', S), ('","durationMs":', R),
             (',"status":"', S), ('"', R),                                   # optional ,"errorMessage":"..." pre-rendered (omitempty)
             ('},"audit":{"inputDataHash":"', S), ('","outputDataHash":"', S), ('","metadata":', R)]
    if with_proof:
        parts += [('}},"proof":{"type":"', S), ('","created":"', S), ('","verificationMethod":"', S), ('","proofPurpose":"', S),
                  ('","proofValue":"', S)]
        tail = '"}}'
    else:
        tail = '}},"proof":' + go_json.vc_proof(go_json.EMPTY_PROOF) + "}"
    return [p[0].encode() for p in parts] + [tail.encode()], [p[1] for p in parts]


def vc_document_values(doc, proof=None):
    """One document's values in the order of vc_document_template (with_proof = proof is not None)."""
    cs = doc["credentialSubject"]
    ex, au, ca, ta = cs["execution"], cs["audit"], cs["caller"], cs["target"]
    u = lambda s: s.encode("utf-8", "surrogatepass") if isinstance(s, str) else bytes(s)
    em = ex.get("errorMessage")
    vals = [go_json.string_list(doc["@context"]).encode(), go_json.string_list(doc["type"]).encode(), u(doc["id"]), u(doc["issuer"]),
            u(doc["issuanceDate"]), u(cs["executionId"]), u(cs["workflowId"]), u(cs["sessionId"]), u(ca["did"]), u(ca["type"]),
            u(ca["agentNodeDid"]), u(ta["did"]), u(ta["agentNodeDid"]), u(ta["functionName"]), u(ex["inputHash"]), u(ex["outputHash"]),
            u(ex["timestamp"]), b"%d" % int(ex["durationMs"]), u(ex["status"]),
            (b',"errorMessage":' + go_json.any_string(em).encode("utf-8")) if em else b"",
            u(au["inputDataHash"]), u(au["outputDataHash"]), go_json.value(au.get("metadata")).encode("utf-8")]
    if proof is not None:
        vals += [u(proof.get("type", "")), u(proof.get("created", "")), u(proof.get("verificationMethod", "")),
                 u(proof.get("proofPurpose", "")), u(proof.get("proofValue", ""))]
    return vals


def workflow_vc_document_template(with_proof=False, ctx=None):
    """Template of json.Marshal(types.WorkflowVCDocument) on the GPU (see workflow_vc_document_template_parts)."""
    return JsonTemplate(*workflow_vc_document_template_parts(with_proof), ctx)


def workflow_vc_document_template_parts(with_proof=False):
    """(segments, kinds) of json.Marshal(types.WorkflowVCDocument) (pkg/types/did_types.go:146-180; signed over a zero Proof at
    internal/services/vc_service.go:686-693, verified the same way at :1589-1597).  componentVcIds ([]string), the two step
    counts (int), the optional endTime (*string, omitempty) and the metadata map are pre-rendered raw values."""
    S, R = STRING, RAW
    parts = [('{"@context":', R), (',"type":', R), (',"id":"', S), ('","issuer":"', S), ('","issuanceDate":"', S),
             ('","credentialSubject":{"workflowId":"', S), ('","sessionId":"', S), ('","componentVcIds":', R), (',"totalSteps":', R),
             (',"completedSteps":', R), (',"status":"', S), ('","startTime":"', S), ('"', R),          # optional ,"endTime":"..."
             (',"snapshotTime":"', S), ('","orchestrator":{"did":"', S), ('","type":"', S), ('","agentNodeDid":"', S),
             ('"},"audit":{"inputDataHash":"', S), ('","outputDataHash":"', S), ('","metadata":', R)]
    if with_proof:
        parts += [('}},"proof":{"type":"', S), ('","created":"', S), ('","verificationMethod":"', S), ('","proofPurpose":"', S),
                  ('","proofValue":"', S)]
        tail = '"}}'
    else:
        tail = '}},"proof":' + go_json.vc_proof(go_json.EMPTY_PROOF) + "}"
    return [p[0].encode() for p in parts] + [tail.encode()], [p[1] for p in parts]


def workflow_vc_document_values(doc, proof=None):
    """One workflow document's values in the order of workflow_vc_document_template."""
    cs = doc["credentialSubject"]
    orc, au = cs["orchestrator"], cs["audit"]
    u = lambda s: s.encode("utf-8", "surrogatepass") if isinstance(s, str) else bytes(s)
    vals = [go_json.string_list(doc["@context"]).encode(), go_json.string_list(doc["type"]).encode(), u(doc["id"]), u(doc["issuer"]),
            u(doc["issuanceDate"]), u(cs["workflowId"]), u(cs["sessionId"]), go_json.string_list(cs["componentVcIds"]).encode("utf-8"),
            b"%d" % int(cs["totalSteps"]), b"%d" % int(cs["completedSteps"]), u(cs["status"]), u(cs["startTime"]),
            (b',"endTime":' + go_json.string(cs["endTime"]).encode("utf-8")) if cs.get("endTime") is not None else b"",
            u(cs["snapshotTime"]), u(orc["did"]), u(orc["type"]), u(orc["agentNodeDid"]), u(au["inputDataHash"]), u(au["outputDataHash"]),
            go_json.value(au.get("metadata")).encode("utf-8")]
    if proof is not None:
        vals += [u(proof.get("type", "")), u(proof.get("created", "")), u(proof.get("verificationMethod", "")),
                 u(proof.get("proofPurpose", "")), u(proof.get("proofValue", ""))]
    return vals


def webhook_payload_template_parts():
    """(segments, kinds) of json.Marshal(types.ExecutionWebhookPayload) (pkg/types/webhook.go:42-53, marshalled at
    internal/services/webhook_dispatcher.go:299): six strings, the omitempty members pre-rendered as one raw value, timestamp."""
    S, R = STRING, RAW
    parts = [('{"event":"', S), ('","execution_id":"', S), ('","workflow_id":"', S), ('","status":"', S), ('","target":"', S), ('","type":"', S),
             ('"', R), (',"timestamp":"', S)]
    return [p[0].encode() for p in parts] + [b'"}'], [p[1] for p in parts]


def webhook_payload_values(p):
    u = lambda s: s.encode("utf-8", "surrogatepass")
    opt = b""
    if p.get("duration_ms") is not None:
        opt += b',"duration_ms":%d' % int(p["duration_ms"])
    if p.get("result") is not None:
        opt += b',"result":' + go_json.value(p["result"]).encode("utf-8")
    if p.get("error_message") is not None:
        opt += b',"error_message":' + go_json.string(p["error_message"]).encode("utf-8")
    return [u(p["event"]), u(p["execution_id"]), u(p["workflow_id"]), u(p["status"]), u(p["target"]), u(p["type"]), opt, u(p["timestamp"])]


def synthetic_stored_vcs_dev(ctx, d_expanded, dids, d_key_index, n, seed=0, str_len=48, audit_columns=False):
    """n stored execution-VC documents of realistic size (~1.3 KB: DIDs, hashes, timestamps; nothing to escape) built on the device
    the way an issuer would: values -> template without proof -> signing bytes -> expanded-key signatures -> base64url ->
    template with proof.  d_expanded: K x 96 expanded keys; dids: their K DIDs (all of one length); d_key_index: n int32 issuer
    indices.  Returns (d_docs uint8, d_doc_off int64 [n+1], d_msgs, d_msg_off, d_sigs) — the signing bytes are those the
    reference verifies, for comparison.  With audit_columns, also (d_cols uint8, d_col_off int64 [n*10+1]): the ExecutionVC
    record written with each document, its _abi.AUDIT_COLUMNS columns packed as afc_vc_audit_stored_batch takes them."""
    import torch
    dev = d_key_index.device
    t0, t1 = vc_document_template(False, ctx), vc_document_template(True, ctx)
    did_len = len(dids[0])
    if any(len(d) != did_len for d in dids):
        raise ValueError("DIDs of one length")
    g = torch.Generator(device=dev); g.manual_seed(seed)
    alphabet = torch.tensor(list(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789-_:"), dtype=torch.uint8, device=dev)
    d_dids = torch.tensor(np.frombuffer(b"".join(d.encode() for d in dids), dtype=np.uint8).reshape(len(dids), did_len).copy(), device=dev)
    const = lambda b: torch.tensor(list(b), dtype=torch.uint8, device=dev).expand(n, len(b))
    rand = lambda w: alphabet[torch.randint(0, alphabet.numel(), (n, w), device=dev, generator=g)]
    issuer = d_dids[d_key_index.long()]
    dur = torch.cat([torch.randint(1, 10, (n, 1), device=dev, generator=g), torch.randint(0, 10, (n, 5), device=dev, generator=g)], 1).to(torch.uint8) + 0x30
    cols = [const(b'["https://www.w3.org/2018/credentials/v1","https://agentfield.example.com/contexts/execution/v1"]'),
            const(b'["VerifiableCredential","AgentFieldExecutionCredential"]'), rand(str_len), issuer, const(b"2026-09-21T06:00:00Z"),
            rand(str_len), rand(str_len), rand(str_len), issuer, const(b"agent"), rand(str_len), rand(str_len), rand(str_len), rand(24),
            rand(43), rand(43), const(b"2026-09-21T06:00:00Z"), dur, const(b"succeeded"), const(b""), rand(43), rand(43),
            const(b'{"agentfield_version":"1.0.0","vc_version":"1.0"}')]

    def packed(columns):
        widths = [c.shape[1] for c in columns]
        rows = torch.cat(columns, 1).contiguous()
        F, row = len(columns), sum(widths)
        starts = torch.tensor(np.concatenate([[0], np.cumsum(widths)[:-1]]), dtype=torch.int64, device=dev)
        off = torch.empty(n * F + 1, dtype=torch.int64, device=dev)
        off[:-1] = (torch.arange(n, device=dev, dtype=torch.int64)[:, None] * row + starts[None, :]).reshape(-1)
        off[-1] = n * row
        return rows.view(-1), off
    vals, voff = packed(cols)
    d_msgs, d_moff = t0.fill_dev(vals, voff, n)
    d_sigs = torch.empty((n, 64), dtype=torch.uint8, device=dev)
    ctx.sign_expanded_dev(d_expanded, d_key_index, d_msgs, d_moff, n, d_sigs)
    d_pv = torch.empty((n, 86), dtype=torch.uint8, device=dev)
    ctx.b64url_encode_dev(d_sigs, 64, n, d_pv)
    cols += [const(b"Ed25519Signature2020"), const(b"2026-09-21T06:00:01Z"), torch.cat([issuer, const(b"#key-1")], 1), const(b"assertionMethod"), d_pv]
    del vals, voff
    vals, voff = packed(cols)
    d_docs, d_doff = t1.fill_dev(vals, voff, n)
    if not audit_columns:
        return d_docs, d_doff, d_msgs, d_moff, d_sigs
    del vals, voff
    # issuer, executionId, workflowId, sessionId, caller.did, target.did, status, inputHash, outputHash, proofValue
    d_cols, d_col_off = packed([cols[k] for k in (3, 5, 6, 7, 8, 11, 18, 14, 15, 27)])
    return d_docs, d_doff, d_msgs, d_moff, d_sigs, d_cols, d_col_off


def synthetic_issue_requests(dids, n, seed=0, payload_bytes=(64, 2048), nil_frac=0.1, err_frac=0.01, long_frac=0.0, long_bytes=256 << 10):
    """n GenerateExecutionVC requests (the dicts of services.VCService.generate_execution_vc_batch) of realistic shape: issuers drawn
    from `dids` in turn, UUID-like ids, RFC 3339 times, input and output payloads of payload_bytes[0]..payload_bytes[1] bytes (uniform,
    seeded; nil_frac of them nil), err_frac of the requests with an error message that needs escaping (a third of those longer than
    500 bytes, cut inside a rune), and long_frac of the payloads long_bytes long.  The payloads are views of one random buffer."""
    rng = np.random.default_rng(seed)
    lo, hi = payload_bytes
    lens = rng.integers(lo, hi + 1, 2 * n)
    lens[rng.random(2 * n) < long_frac] = long_bytes
    nil = rng.random(2 * n) < nil_frac
    starts = rng.integers(0, 4096, 2 * n)
    pool = memoryview(rng.integers(0, 256, int(lens.max()) + 4096, dtype=np.uint8).tobytes())
    errs = np.flatnonzero(rng.random(n) < err_frac)
    err_text = {}
    for j, i in enumerate(errs):
        base = 'tool "fetch" failed: <status 502> & retry\n\tline 2   ' + "é中\U0001F600" * int(rng.integers(1, 8))
        err_text[int(i)] = base * (40 if j % 3 == 0 else 1)
    statuses = ("succeeded", "failed", "running", "completed", "timeout")
    out = []
    for i in range(n):
        did = dids[i % len(dids)]
        p = [None if nil[2 * i + k] else pool[int(starts[2 * i + k]):int(starts[2 * i + k] + lens[2 * i + k])] for k in (0, 1)]
        out.append({"vc_id": "%08x-4e7a-4b1c-9d2e-%012x" % (i, i * 2654435761 % (1 << 48)), "caller_did": did,
                    "issuance_date": "2026-09-21T06:%02d:%02dZ" % (i // 60 % 60, i % 60), "execution_id": "exec_%016x" % i,
                    "workflow_id": "wf_%08x" % (i // 16), "session_id": "sess_%06x" % (i // 256), "caller_type": "agent",
                    "agent_node_did": dids[(i + 1) % len(dids)], "target_did": dids[(i + 7) % len(dids)], "function_name": "tool.fetch_%d" % (i % 97),
                    "input": p[0], "output": p[1], "status": statuses[i % len(statuses)], "error_message": err_text.get(i, ""),
                    "duration_ms": int(rng.integers(0, 10 ** 7)), "timestamp": "2026-09-21T05:59:%02d.%06dZ" % (i % 60, i % 1000000),
                    "proof_created": "2026-09-21T06:00:01Z"})
    return out
