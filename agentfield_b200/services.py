"""Host-side mirror of the reference's service-level seams for this path, batched (SURVEY.md §8a rows D1, E1, E2, H1, W1):

    VCService.hashData / signVC / verifyVCSignature / GenerateExecutionVC / VerifyVC
        control-plane/internal/services/vc_service.go:138-239, 242-289, 434-515
    generateWorkflowVCDocument / createWorkflowVCDocument / signWorkflowVC / determineWorkflowStatus / countCompletedSteps
        control-plane/internal/services/vc_service.go:525-787
    VerifyWorkflowVCComprehensive / performIntegrityChecks / performSecurityAnalysis / performComplianceChecks /
    verifyWorkflowVCSignature / calculateOverallScore
        control-plane/internal/services/vc_service.go:1037-1383, 1386-1644; pkg/types/status.go:28-75
    generateWebhookSignature
        control-plane/internal/services/webhook_dispatcher.go:470-474

Same names (snake_cased) and behaviour; each takes a BATCH (the natural seam is the loop in
VerifyWorkflowVCComprehensive, vc_service.go:1442-1512, or a linger queue in front of one-per-request calls) and does
every hash / signature on the GPU through the C ABI.  The canonical JSON bytes come from go_json.py on the host or, with
canonical_on_device=True, from the device: GenerateExecutionVC's hashes, documents and signatures in one call (afc_vc_issue_execution_batch).
"""
import base64
import datetime
import json

import numpy as np

from . import _abi, go_json
from .crypto import Hasher, MAC, default_context, pack, pack32
from .identity import ExpandedKeys, KeySet, public_jwk


def _b64url(b: bytes) -> str:
    return base64.urlsafe_b64encode(b).rstrip(b"=").decode()


def _b64url_decode(s: str) -> bytes:
    return base64.urlsafe_b64decode(s + "=" * (-len(s) % 4))


def marshal_data_or_null(data):
    """vc_service.go:1298-1306 — json.Marshal([]byte): nil -> null, else the std-base64 text in quotes."""
    if data is None:
        return b"null"
    return b'"' + base64.b64encode(data) + b'"'


_STATUS_CANONICAL = {"unknown", "pending", "queued", "running", "succeeded", "failed", "cancelled", "timeout"}
_STATUS_ALIASES = {"success": "succeeded", "successful": "succeeded", "completed": "succeeded", "complete": "succeeded", "done": "succeeded",
                   "ok": "succeeded", "error": "failed", "failure": "failed", "errored": "failed", "canceled": "cancelled", "cancel": "cancelled",
                   "timed_out": "timeout", "wait": "queued", "waiting": "queued", "in_progress": "running", "processing": "running"}


def normalize_execution_status(status: str) -> str:
    """types.NormalizeExecutionStatus (pkg/types/status.go:51-63)."""
    s = status.strip().lower()
    if not s:
        return "unknown"
    if s in _STATUS_CANONICAL:
        return s
    return _STATUS_ALIASES.get(s, "unknown")


def is_terminal_execution_status(status: str) -> bool:
    return normalize_execution_status(status) in ("succeeded", "failed", "cancelled", "timeout")


def determine_workflow_status(execution_vcs) -> str:
    """determineWorkflowStatus (vc_service.go:721-772): the worst state present wins."""
    if not execution_vcs:
        return "pending"
    seen = {normalize_execution_status(v["status"]) for v in execution_vcs}
    for s in ("failed", "timeout", "cancelled", "running", "queued", "pending", "unknown"):
        if s in seen:
            return s
    return "succeeded"


def count_completed_steps(execution_vcs) -> int:
    return sum(1 for v in execution_vcs if normalize_execution_status(v["status"]) == "succeeded")


_STATUS_NAMES = ("unknown", "pending", "queued", "running", "succeeded", "failed", "cancelled", "timeout")     # AFC_WORKFLOW summary[0]
_NO_RECORD = 0xFFFFFFFF


def _rfc3339(t) -> str:
    """time.Time.UTC().Format(time.RFC3339) of an aware datetime."""
    u = t.astimezone(datetime.timezone.utc)
    return "%04d-%02d-%02dT%02d:%02d:%02dZ" % (u.year, u.month, u.day, u.hour, u.minute, u.second)


def create_workflow_vc_document(workflow_id, session_id, component_vc_ids, status, start_time, end_time, issuer_did, vc_id, issuance_date,
                                snapshot_time):
    """createWorkflowVCDocument (vc_service.go:635-683).  Times are RFC 3339 strings (the reference formats time.Time with
    UTC().Format(time.RFC3339)); vc_id / issuance_date / snapshot_time are inputs here where the reference reads the clock."""
    n = len(component_vc_ids) if component_vc_ids is not None else 0
    cs = {"workflowId": workflow_id, "sessionId": session_id, "componentVcIds": component_vc_ids, "totalSteps": n, "completedSteps": n,
          "status": status, "startTime": start_time, "endTime": end_time, "snapshotTime": snapshot_time,
          "orchestrator": {"did": issuer_did, "type": "agentfield_server", "agentNodeDid": issuer_did},
          "audit": {"inputDataHash": "", "outputDataHash": "",
                    "metadata": {"agentfield_version": "1.0.0", "vc_version": "1.0", "workflow_type": "agent_execution_chain",
                                 "total_executions": n}}}
    return {"@context": ["https://www.w3.org/2018/credentials/v1", "https://agentfield.example.com/contexts/workflow/v1"],
            "type": ["VerifiableCredential", "AgentFieldWorkflowCredential"],
            "id": "urn:agentfield:workflow-vc:%s" % vc_id, "issuer": issuer_did, "issuanceDate": issuance_date, "credentialSubject": cs}


def generate_webhook_signature_batch(secrets, bodies, ctx=None):
    """generateWebhookSignature for many deliveries: "sha256=" + hex(HMAC-SHA256(secret, body))."""
    tags = MAC(ctx or default_context()).hmac_sha256_batch([s.encode() if isinstance(s, str) else s for s in secrets], bodies)
    return ["sha256=" + t.hex() for t in tags]


def _wh_bytes(v):
    return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)


def pack_webhook_deliveries(records):
    """The packed inputs of afc_webhook_sign_batch (include/afcrypto.h) for records as build_webhook_payload takes them, plus an
    optional "secret" (str or bytes; None = the webhook has none)."""
    cols, flags, dur, results, secrets = [], [], [], [], []
    for r in records:
        cols += [_wh_bytes(r[k]) if k != "error_message" else _wh_bytes(r.get(k) or b"") for k in _abi.WEBHOOK_COLUMNS]
        f = 0
        if r.get("duration_ms") is not None:
            f |= _abi.WEBHOOK_HAS_DURATION
        if r.get("error_message") is not None:
            f |= _abi.WEBHOOK_HAS_ERROR_MESSAGE
        if r.get("secret") is not None:
            f |= _abi.WEBHOOK_HAS_SECRET
        flags.append(f)
        dur.append(int(r["duration_ms"]) if r.get("duration_ms") is not None else 0)
        results.append(bytes(r.get("result") or b""))
        secrets.append(_wh_bytes(r["secret"]) if r.get("secret") is not None else b"")
    cb, co = pack(cols)
    rb, ro = pack(results)
    sb, so = pack32(secrets)
    return cb, co, np.array(dur, dtype=np.int64), np.array(flags, dtype=np.uint8), rb, ro, sb, so


def sign_webhook_delivery_host(record):
    """One delivery built on the host (the AFC_WEBHOOK_HOST path): {"body", "header"}."""
    import hashlib
    import hmac
    body = go_json.build_webhook_payload(record)
    sec = record.get("secret")
    return {"body": body, "header": None if sec is None else "sha256=" + hmac.new(_wh_bytes(sec), body, hashlib.sha256).hexdigest()}


def sign_webhook_deliveries_batch(records, ctx=None):
    """determineWebhookEvent + buildPayload + json.Marshal + generateWebhookSignature (webhook_dispatcher.go:294-320) for many
    deliveries in one device call: [{"body": bytes, "header": str | None}].  Deliveries the device declines (AFC_WEBHOOK_HOST) are
    built by the host mirror."""
    if not records:
        return []
    ctx = ctx or default_context()
    bodies, off, headers, status = ctx.webhook_sign_packed(*pack_webhook_deliveries(records))
    out = []
    for i, r in enumerate(records):
        if status[i] == _abi.WEBHOOK_HOST:
            out.append(sign_webhook_delivery_host(r))
            continue
        out.append({"body": bytes(bodies[int(off[i]):int(off[i + 1])]),
                    "header": headers[i].tobytes().decode() if r.get("secret") is not None else None})
    return out


class VCService:
    """Batched issue / verify of execution VCs over a key cache (DID -> expanded key) and an issuer key set."""

    def __init__(self, keys: ExpandedKeys, ctx=None, hash_sensitive_data=True, canonical_on_device=False, store=None):
        self.ctx = ctx or keys.ctx
        self.keys = keys
        self.store = store                                        # vc_store.ExecutionVCStore: the issued batch is persisted in ONE transaction
        self.hash_sensitive_data = hash_sensitive_data
        self.canonical_on_device = canonical_on_device
        self._keyset = None
        self._keyset_dids = None

    # -- H1
    def hash_data_batch(self, datas):
        if not self.hash_sensitive_data:
            return [""] * len(datas)
        return [_b64url(d) for d in Hasher(self.ctx).sha256_batch(datas)]

    # -- E1 / D1
    def generate_execution_vc_batch(self, requests, log=None):
        """requests: dicts with execution_id, workflow_id, session_id, caller_did, target_did, agent_node_did, caller_type,
        function_name, input (bytes|None), output (bytes|None), status, error_message (str|None), duration_ms, timestamp,
        vc_id, issuance_date, proof_created.  Returns [{"vc_document": bytes, "signature": str, "input_hash", "output_hash"}].
        With canonical_on_device the hashes, documents and signatures come from one device call (ExpandedKeys.issue).  log: an
        audit.Auditor that receives the stored documents, in batch order."""
        n = len(requests)
        issued = self.keys.issue(requests, self.hash_sensitive_data, log) if self.canonical_on_device and n else None
        if issued is None:
            hashes = self.hash_data_batch([marshal_data_or_null(r.get("input")) for r in requests] +
                                          [marshal_data_or_null(r.get("output")) for r in requests])
        else:
            hashes = [v["input_hash"] for v in issued] + [v["output_hash"] for v in issued]
        docs, msgs = [], []
        for i, r in enumerate(requests):
            ih, oh = hashes[i], hashes[n + i]
            em = go_json.truncate_error_message(r.get("error_message"))                 # vc_service.go:153-160 (bytes, not runes)
            doc = {
                "@context": ["https://www.w3.org/2018/credentials/v1", "https://agentfield.example.com/contexts/execution/v1"],
                "type": ["VerifiableCredential", "AgentFieldExecutionCredential"],
                "id": "urn:agentfield:vc:%s" % r["vc_id"], "issuer": r["caller_did"], "issuanceDate": r["issuance_date"],
                "credentialSubject": {
                    "executionId": r["execution_id"], "workflowId": r["workflow_id"], "sessionId": r["session_id"],
                    "caller": {"did": r["caller_did"], "type": r.get("caller_type", "agent"), "agentNodeDid": r["agent_node_did"]},
                    "target": {"did": r.get("target_did", ""), "agentNodeDid": r["agent_node_did"], "functionName": r.get("function_name", "")},
                    "execution": {"inputHash": ih, "outputHash": oh, "timestamp": r["timestamp"], "durationMs": r["duration_ms"],
                                  "status": r["status"], "errorMessage": em or ""},
                    "audit": {"inputDataHash": ih, "outputDataHash": oh, "metadata": {"agentfield_version": "1.0.0", "vc_version": "1.0"}},
                },
            }
            docs.append(doc)
            if issued is None:
                msgs.append(go_json.vc_document(doc))                                    # zero-valued proof: what signVC signs
        if issued is None:
            pvs = [_b64url(sig) for sig in self.keys.sign_batch([r["caller_did"] for r in requests], msgs)]      # one GPU batch
        else:
            pvs = [v["signature"] for v in issued]
        proofs = [{"type": "Ed25519Signature2020", "created": r["proof_created"], "verificationMethod": "%s#key-1" % r["caller_did"],
                   "proofPurpose": "assertionMethod", "proofValue": pv} for r, pv in zip(requests, pvs)]
        if issued is None:
            stored = [go_json.vc_document(d, p) for d, p in zip(docs, proofs)]
            if log is not None and stored:
                log.append(stored)
        else:
            stored = [v["vc_document"] for v in issued]
        out = []
        for doc, proof, vc_bytes in zip(docs, proofs, stored):
            out.append({"vc_document": vc_bytes, "signature": proof["proofValue"],
                        "input_hash": doc["credentialSubject"]["execution"]["inputHash"],
                        "output_hash": doc["credentialSubject"]["execution"]["outputHash"], "doc": doc, "proof": proof})
        if self.store is not None and out:                        # vc_service.go:229-233, for the whole batch at once (group commit)
            self.store.store_execution_vcs([
                {"vc_id": r["vc_id"], "execution_id": r["execution_id"], "workflow_id": r["workflow_id"], "session_id": r["session_id"],
                 "issuer_did": r["caller_did"], "target_did": r.get("target_did", ""), "caller_did": r["caller_did"], "vc_document": v["vc_document"],
                 "signature": v["signature"], "input_hash": v["input_hash"], "output_hash": v["output_hash"],
                 "status": normalize_execution_status(r["status"])} for r, v in zip(requests, out)])
        return out

    # -- E2 / D1
    def verify_vc_batch(self, vcs):
        """VerifyVC for many stored documents: re-marshal the parsed document with a zero proof, resolve the issuer key from
        the cache, one keyed GPU verification batch.  vcs: the dicts returned by generate_execution_vc_batch (doc + proof)."""
        dids = [v["doc"]["issuer"] for v in vcs]
        uniq = sorted(set(dids))
        if self._keyset is None or self._keyset_dids != uniq:
            if self._keyset is not None:
                self._keyset.close()
            self._keyset = KeySet([self.keys.public_key(d) for d in uniq], self.ctx)
            self._keyset_dids = uniq
        pos = {d: i for i, d in enumerate(uniq)}
        msgs = [go_json.vc_document(v["doc"]) for v in vcs]
        sigs_raw = [_b64url_decode(v["proof"]["proofValue"]) for v in vcs]
        bad = [len(s) != 64 for s in sigs_raw]
        sg = np.zeros((len(vcs), 64), dtype=np.uint8)
        for i, s in enumerate(sigs_raw):
            if not bad[i]:
                sg[i] = np.frombuffer(s, dtype=np.uint8)
        buf, off = pack(msgs)
        ok = self._keyset.verify_packed(np.array([pos[d] for d in dids], dtype=np.uint32), sg, buf, off)
        return [bool(o) and not b for o, b in zip(ok, bad)]

    # -- workflow-level credentials (vc_service.go:525-718)
    def generate_workflow_vc_batch(self, workflows):
        """generateWorkflowVCDocument for many workflows, all signatures in one GPU batch.  Each workflow: workflow_id,
        execution_vcs (the ExecutionVC records: vc_id, session_id, status, created_at (RFC 3339, UTC), issuer_did), root_did (the
        issuer when the workflow has no execution VCs), vc_id, workflow_vc_id, issuance_date, snapshot_time, proof_created.
        Returns WorkflowVC-shaped dicts (pkg/types/did_types.go:88-104) plus "doc" / "proof"."""
        docs, metas = [], []
        for w in workflows:
            evs = w["execution_vcs"]
            status = determine_workflow_status(evs)
            ids = [v["vc_id"] for v in evs]
            session_id = evs[0]["session_id"] if evs else ""
            if evs:
                times = [v["created_at"] for v in evs]                # RFC 3339 in UTC with equal precision sorts chronologically
                start, latest = min(times), max(times)
                end = latest if is_terminal_execution_status(status) else None
                issuer = evs[0]["issuer_did"]
            else:
                start, end, issuer = w["snapshot_time"], None, w["root_did"]
            doc = create_workflow_vc_document(w["workflow_id"], session_id, ids, status, start, end, issuer, w["vc_id"], w["issuance_date"],
                                              w["snapshot_time"])
            docs.append(doc)
            metas.append((w, evs, status, ids, session_id, start, end, issuer))
        sigs = self.keys.sign_batch([m[7] for m in metas], [go_json.workflow_vc_document(d) for d in docs])   # signWorkflowVC: zero proof
        out = []
        for doc, (w, evs, status, ids, session_id, start, end, issuer), sig in zip(docs, metas, sigs):
            proof = {"type": "Ed25519Signature2020", "created": w["proof_created"], "verificationMethod": "%s#key-1" % issuer,
                     "proofPurpose": "assertionMethod", "proofValue": _b64url(sig)}
            vc_bytes = go_json.workflow_vc_document(doc, proof)
            out.append({"workflow_id": w["workflow_id"], "session_id": session_id, "component_vcs": ids, "workflow_vc_id": w["workflow_vc_id"],
                        "status": status, "start_time": start, "end_time": end, "total_steps": len(evs),
                        "completed_steps": count_completed_steps(evs), "vc_document": vc_bytes, "signature": proof["proofValue"],
                        "issuer_did": issuer, "snapshot_time": w["snapshot_time"], "storage_uri": "", "document_size_bytes": len(vc_bytes),
                        "doc": doc, "proof": proof})
        return out

    def issue_workflow_vc_batch(self, workflows):
        """generate_workflow_vc_batch in one device call (ExpandedKeys.issue_workflows): the same inputs, except that each record's
        created_at is an aware datetime, and the same WorkflowVC-shaped dicts without "doc" / "proof".  Workflows the device declines
        (AFC_WORKFLOW_HOST: a status that is not printable ASCII) go through generate_workflow_vc_batch."""
        if not workflows:
            return []
        issued = self.keys.issue_workflows(workflows)
        host = [i for i, v in enumerate(issued) if v["state"] == _abi.WORKFLOW_HOST]
        by_host = {}
        if host:
            text = [dict(workflows[i], execution_vcs=[dict(v, created_at=_rfc3339(v["created_at"])) for v in workflows[i]["execution_vcs"]])
                    for i in host]
            for i, v in zip(host, self.generate_workflow_vc_batch(text)):
                del v["doc"], v["proof"]
                by_host[i] = v
        out = []
        for i, (w, v) in enumerate(zip(workflows, issued)):
            if i in by_host:
                out.append(by_host[i])
                continue
            evs = w["execution_vcs"]
            status, completed, start, end = v["summary"]
            vc_bytes = v["vc_document"]
            out.append({"workflow_id": w["workflow_id"], "session_id": evs[0]["session_id"] if evs else "", "component_vcs": [e["vc_id"] for e in evs],
                        "workflow_vc_id": w["workflow_vc_id"], "status": _STATUS_NAMES[status],
                        "start_time": _rfc3339(evs[start]["created_at"]) if evs else w["snapshot_time"],
                        "end_time": _rfc3339(evs[end]["created_at"]) if end != _NO_RECORD else None, "total_steps": len(evs),
                        "completed_steps": completed, "vc_document": vc_bytes, "signature": v["signature"], "issuer_did": self.keys.workflow_issuer(w),
                        "snapshot_time": w["snapshot_time"], "storage_uri": "", "document_size_bytes": len(vc_bytes)})
        return out

    # -- workflow VC chains (vc_service.go:292-338, 810-870; internal/handlers/ui/did.go:383)
    def get_workflow_vc_chain_batch(self, workflows, directory):
        """GetWorkflowVCChain + c.JSON for many workflows, in request order: each body is the bytes the chain endpoint writes.  Each
        workflow: the inputs of issue_workflow_vc_batch with complete ExecutionVC records (ExpandedKeys.pack_chain_requests), plus
        workflow_vc_id, resolved_at and snapshot (an aware datetime).  directory: an identity.DIDDirectory (DIDService.did_directory).
        One device call (ExpandedKeys.workflow_chains); workflows it declines (AFC_CHAIN_HOST) are built by the host mirror,
        workflow_chain_body over issue_workflow_vc_batch's output, which raises ValueError where json.Marshal fails in Go."""
        if not workflows:
            return []
        res = self.keys.workflow_chains(workflows, directory)
        out = [body for _, body in res]
        host = [i for i, (st, _) in enumerate(res) if st == _abi.CHAIN_HOST]
        if host:
            keys = dict(zip(directory.dids, directory.pks))
            for i, wvc in zip(host, self.issue_workflow_vc_batch([workflows[i] for i in host])):
                out[i] = workflow_chain_body(workflows[i], wvc, keys)
        return out

    def _keyed_verify(self, dids, msgs, proof_values):
        """ed25519.Verify for many (issuer DID, canonical bytes, base64url signature) through one keyed GPU batch.  A DID the
        cache cannot resolve or a signature that does not decode gives None (the reference reports those as errors, not False)."""
        known = [d in self.keys._index for d in dids]
        uniq = sorted({d for d, k in zip(dids, known) if k})
        if self._keyset is None or self._keyset_dids != uniq:
            if self._keyset is not None:
                self._keyset.close()
            self._keyset = KeySet([self.keys.public_key(d) for d in uniq], self.ctx) if uniq else None
            self._keyset_dids = uniq
        pos = {d: i for i, d in enumerate(uniq)}
        sg = np.zeros((len(dids), 64), dtype=np.uint8)
        state = []
        for i, (d, k, pv) in enumerate(zip(dids, known, proof_values)):
            try:
                raw = _b64url_decode_strict(pv)
            except ValueError:
                state.append("bad_encoding"); continue
            if not k:
                state.append("unresolved"); continue
            if len(raw) != 64:
                state.append("bad_length"); continue            # ed25519.Verify: plain false
            sg[i] = np.frombuffer(raw, dtype=np.uint8); state.append("ok")
        if not uniq:
            return [None if st in ("unresolved", "bad_encoding") else False for st in state]
        buf, off = pack(msgs)
        ki = np.array([pos.get(d, 0) for d in dids], dtype=np.uint32)
        ok = self._keyset.verify_packed(ki, sg, buf, off)
        return [bool(o) if st == "ok" else (False if st == "bad_length" else None) for o, st in zip(ok, state)]

    def verify_workflow_vc_batch(self, workflow_vcs):
        """verifyWorkflowVCSignature (vc_service.go:1589-1625) for many stored workflow VCs: parse, zero the proof, re-marshal
        (metadata numbers come back as float64), verify against the issuer's key."""
        import json
        docs = [json.loads(w["vc_document"], parse_int=float) for w in workflow_vcs]
        for d in docs:
            d["credentialSubject"]["audit"]["metadata"] = go_json.unmarshal_numbers(d["credentialSubject"]["audit"].get("metadata"))
        res = self._keyed_verify([d["issuer"] for d in docs], [go_json.workflow_vc_document(d) for d in docs],
                                 [d["proof"]["proofValue"] for d in docs])
        return [bool(r) for r in res]

    # -- stored documents verified on the device (afc_vc_verify_stored_batch)
    def verify_stored_vc_batch(self, stored_docs):
        """VerifyVC (vc_service.go:242-289) for many stored execution-VC documents (bytes as stored): one VCVerificationResponse-shaped
        dict per document (valid, error, message, issuer_did, issued_at; "" where Go omits the field).  Documents in the exact form
        json.Marshal writes are parsed, re-assembled and verified on the GPU; only the others are parsed and re-marshalled here."""
        return self._verify_stored(_abi.DOC_EXECUTION_VC, stored_docs)

    def verify_stored_workflow_vc_batch(self, stored_docs):
        """The same for stored workflow-VC documents (verifyWorkflowVCSignature, vc_service.go:1589-1625)."""
        return self._verify_stored(_abi.DOC_WORKFLOW_VC, stored_docs)

    def _named_keyset(self):
        dids = sorted(self.keys._index)
        if getattr(self, "_stored_keyset", None) is None or self._stored_keyset_dids != dids:
            if getattr(self, "_stored_keyset", None) is not None:
                self._stored_keyset.close()
            self._stored_keyset = KeySet([self.keys.public_key(d) for d in dids], self.ctx, dids=dids) if dids else None
            self._stored_keyset_dids = dids
        return self._stored_keyset

    # -- documents in any JSON spelling verified on the device (afc_vc_verify_json_batch)
    def verify_vc_json_batch(self, raw_docs):
        """VerifyVC(json.RawMessage) (vc_service.go:242-289) for many execution-VC documents as clients send them: request bodies of
        POST /api/v1/did/verify and files given to `af vc verify`, in any JSON spelling.  Returns what verify_stored_vc_batch returns;
        the spellings real clients produce are re-marshalled and verified on the GPU, only the others here."""
        return self._verify_stored(_abi.DOC_EXECUTION_VC, raw_docs, json_spelling=True)

    def verify_workflow_vc_json_batch(self, raw_docs):
        """The same for workflow-VC documents (verifyWorkflowVCSignature, vc_service.go:1589-1625)."""
        return self._verify_stored(_abi.DOC_WORKFLOW_VC, raw_docs, json_spelling=True)

    def _verify_stored(self, kind, stored_docs, json_spelling=False):
        """json_spelling: the device call re-marshals documents in any spelling (afc_vc_verify_json_batch); it declines invalid UTF-8,
        so the spans of the documents it accepts decode exactly as Go decodes them."""
        docs = [bytes(d) for d in stored_docs]
        n = len(docs)
        ks = self._named_keyset()
        if ks is not None and n:
            status, fields = (ks.verify_json if json_spelling else ks.verify_stored)(kind, docs)
        else:
            status, fields = np.full(n, _abi.VC_HOST, dtype=np.uint8), np.zeros((n, 4), dtype=np.uint32)
        out = [None] * n
        host = []
        for i, (raw, st) in enumerate(zip(docs, status)):
            if st == _abi.VC_VALID:
                iss = raw[fields[i, 0]:fields[i, 0] + fields[i, 1]].decode("utf-8")
                date = json.loads(b'"' + raw[fields[i, 2]:fields[i, 2] + fields[i, 3]] + b'"')
                out[i] = _vc_response(True, message="VC verified successfully", issuer_did=iss, issued_at=date)
            elif st == _abi.VC_INVALID:
                out[i] = _vc_response(False, message="Invalid signature")
            elif st == _abi.VC_UNRESOLVED:
                iss = raw[fields[i, 0]:fields[i, 0] + fields[i, 1]].decode("utf-8")
                out[i] = _vc_response(False, error="failed to resolve issuer DID: DID not found: %s" % iss)
            elif st == _abi.VC_BAD_ENCODING:
                pv = json.loads(raw)["proof"]["proofValue"]
                out[i] = _vc_response(False, error="failed to verify signature: failed to decode signature: illegal base64 data at input byte %d"
                                      % _b64url_error_at(pv))
            else:
                host.append(i)
        # the documents the device declined: today's path (Unmarshal -> Marshal with a zero proof -> keyed verify), batched
        parsed = []
        for i in host:
            try:
                parsed.append((i, go_unmarshal_vc(docs[i], kind)))
            except ValueError as ex:
                out[i] = _vc_response(False, error="failed to parse VC document: %s" % ex)
        if parsed:
            marshal = go_json.vc_document if kind == _abi.DOC_EXECUTION_VC else go_json.workflow_vc_document
            verdicts = self._keyed_verify([d["issuer"] for _, d in parsed], [marshal(d) for _, d in parsed],
                                          [d["proof"]["proofValue"] for _, d in parsed])
            for (i, d), v in zip(parsed, verdicts):
                if v is None and d["issuer"] not in self.keys._index:
                    out[i] = _vc_response(False, error="failed to resolve issuer DID: DID not found: %s" % d["issuer"])
                elif v is None:
                    out[i] = _vc_response(False, error="failed to verify signature: failed to decode signature: illegal base64 data at input byte %d"
                                          % _b64url_error_at(d["proof"]["proofValue"]))
                elif v:
                    out[i] = _vc_response(True, message="VC verified successfully", issuer_did=d["issuer"], issued_at=d["issuanceDate"])
                else:
                    out[i] = _vc_response(False, message="Invalid signature")
        return out

    # -- verification requests answered on the device (afc_vc_verify_request_batch)
    def serve_verify_requests(self, bodies):
        """POST /api/v1/did/verify (did_handlers.go:97-111) for many raw request bodies: (http status, response bytes) per body, the bytes
        c.JSON writes.  Bind, verify and response are built on the GPU in one call; the requests it leaves to the host (AFC_VREQ_HOST) run
        the handler here: the body bound with Go's rules, go_unmarshal_vc's decoding of the document and _keyed_verify."""
        bodies = [bytes(b) for b in bodies]
        ks = self._named_keyset()
        res = ks.verify_requests(bodies) if ks is not None and bodies else [(_abi.VREQ_HOST, b"")] * len(bodies)
        out = []
        for raw, (st, body) in zip(bodies, res):
            if st == _abi.VREQ_HOST:
                out.append(self._verify_request_host(raw))
            else:
                out.append((400 if st == _abi.VREQ_BAD_REQUEST else 200, body))
        return out

    def _verify_request_host(self, raw):
        """One request body through the handler on the host: ShouldBindJSON, VerifyVC, c.JSON."""
        try:
            v = _bind_verify_request(raw)
        except ValueError:
            return 400, b'{"error":"Invalid request body"}'
        if v is _ABSENT:
            return 200, _response_bytes(_vc_response(False, error="failed to parse VC document: unexpected end of JSON input"))
        if v is None:
            d = _zero(_VC_DOC)                            # json.Unmarshal of null leaves the zero document
        elif not isinstance(v, _Obj):
            what = "string" if isinstance(v, str) else "bool" if isinstance(v, bool) else "array" if isinstance(v, list) else "number"
            return 200, _response_bytes(_vc_response(
                False, error="failed to parse VC document: json: cannot unmarshal %s into Go value of type types.VCDocument" % what))
        else:
            try:
                d = _go_into(v, _VC_DOC, _zero(_VC_DOC))
            except ValueError as ex:
                return 200, _response_bytes(_vc_response(False, error="failed to parse VC document: %s" % ex))
        if d["issuer"] not in self.keys._index:
            return 200, _response_bytes(_vc_response(False, error="failed to resolve issuer DID: DID not found: %s" % d["issuer"]))
        pv = d["proof"]["proofValue"]
        v = self._keyed_verify([d["issuer"]], [go_json.vc_document(d)], [pv])[0]
        if v is None:
            r = _vc_response(False, error="failed to verify signature: failed to decode signature: illegal base64 data at input byte %d"
                             % _b64url_error_at(pv))
        elif v:
            r = _vc_response(True, message="VC verified successfully", issuer_did=d["issuer"], issued_at=d["issuanceDate"])
        else:
            r = _vc_response(False, message="Invalid signature")
        return 200, _response_bytes(r)

    # -- comprehensive audit (vc_service.go:926-1005, 1008-1359, 1386-1644)
    def _audit_component(self, ev, doc, verdict, integrity, security, compliance):
        """The checks of one execution VC against its record (performIntegrityChecks, performSecurityAnalysis with
        detectTamperEvidence, performComplianceChecks; vc_service.go:1008-1359), added to the three running results.  doc: the parsed
        document (_parse_execution_doc); verdict: its signature check as _keyed_verify reports it (True, False, or None when the
        issuer does not resolve or proofValue does not decode).  Nothing is verified here."""
        cs, ex = doc["credentialSubject"], doc["credentialSubject"]["execution"]
        ic_issues, tamper = [], []
        pairs = (("issuer_mismatch", "metadata_consistency", "issuer_did", ev["issuer_did"], doc["issuer"], "Issuer DID"),
                 ("execution_id_mismatch", "field_consistency", "execution_id", ev["execution_id"], cs["executionId"], "Execution ID"),
                 ("workflow_id_mismatch", "field_consistency", "workflow_id", ev["workflow_id"], cs["workflowId"], "Workflow ID"),
                 ("session_id_mismatch", "field_consistency", "session_id", ev["session_id"], cs["sessionId"], "Session ID"),
                 ("caller_did_mismatch", "field_consistency", "caller_did", ev["caller_did"], cs["caller"]["did"], "Caller DID"),
                 ("target_did_mismatch", "field_consistency", "target_did", ev["target_did"], cs["target"]["did"], "Target DID"))
        for kind, flag, field, want, got, label in pairs:
            if want != got:
                integrity[flag] = False
                ic_issues.append(_issue(kind, "critical", ev["vc_id"], "%s mismatch between metadata and VC document" % label, field, want, got))
        if normalize_execution_status(ev["status"]) != normalize_execution_status(ex["status"]):
            integrity["field_consistency"] = False
            ic_issues.append(_issue("status_mismatch", "critical", ev["vc_id"], "Status mismatch between metadata and VC document", "status", ev["status"],
                                    ex["status"]))
        for kind, field, want, got, label in (("input_hash_mismatch", "input_hash", ev["input_hash"], ex["inputHash"], "Input hash"),
                                              ("output_hash_mismatch", "output_hash", ev["output_hash"], ex["outputHash"], "Output hash")):
            if want != got:
                integrity["hash_validation"] = False
                ic_issues.append(_issue(kind, "critical", ev["vc_id"], "%s mismatch between metadata and VC document" % label, field, want, got))
        if ev["signature"] != doc["proof"]["proofValue"]:
            integrity["structural_integrity"] = False
            ic_issues.append(_issue("signature_mismatch", "critical", ev["vc_id"], "Signature mismatch between metadata and VC document", "signature",
                                    ev["signature"], doc["proof"]["proofValue"]))
        if not _is_rfc3339(doc["issuanceDate"]):
            integrity["timestamp_validation"] = False
            ic_issues.append(_issue("invalid_timestamp", "critical", ev["vc_id"], "Invalid timestamp", "issuance_date"))
        missing = next((name for name, v in (("@context", doc.get("@context")), ("type", doc.get("type")), ("id", doc.get("id")),
                                             ("issuer", doc.get("issuer")), ("issuanceDate", doc.get("issuanceDate"))) if not v), None)
        if missing:
            integrity["structural_integrity"] = False
            ic_issues.append(_issue("invalid_structure", "critical", ev["vc_id"], "Invalid VC structure: missing %s" % missing))
        integrity["issues"] += ic_issues
        score = 100.0
        if verdict is None and doc["issuer"] not in self.keys._index:
            security["did_authenticity"] = False; score -= 50.0
            security["issues"].append(_issue("did_resolution_failed", "critical", ev["vc_id"], "Failed to resolve issuer DID"))
        elif not verdict:
            security["key_validation"] = False; score -= 40.0
            security["issues"].append(_issue("signature_verification_failed", "critical", ev["vc_id"], "Signature verification failed"))
        if ev["issuer_did"] != doc["issuer"]:
            tamper.append("issuer_did_inconsistency")
        if ev["execution_id"] != cs["executionId"]:
            tamper.append("execution_id_inconsistency")
        if ev["signature"] != doc["proof"]["proofValue"]:
            tamper.append("signature_inconsistency")
        if tamper:
            score -= 20.0
            security["tamper_evidence"] += tamper
            security["issues"].append(_issue("tamper_evidence", "warning", ev["vc_id"], "Tamper evidence detected: %s" % tamper))
        security["security_score"] = min(security["security_score"], score)
        if "https://www.w3.org/2018/credentials/v1" not in (doc.get("@context") or []):
            compliance["w3c_compliance"] = False
            compliance["issues"].append(_issue("w3c_compliance_failure", "warning", doc.get("id", ""), "VC does not meet W3C standards"))
        if not {"VerifiableCredential", "AgentFieldExecutionCredential"} <= set(doc.get("type") or []):
            compliance["agentfield_standard_compliance"] = False
            compliance["issues"].append(_issue("agentfield_compliance_failure", "warning", doc.get("id", ""),
                                               "VC does not meet AgentField standard requirements"))

    def _audit_workflow_vc(self, wf, wf_doc, verdict, security, compliance):
        """The workflow VC's part of VerifyWorkflowVCComprehensive (vc_service.go:1515-1567, checkWorkflowVCCompliance :1628-1644)."""
        if verdict is None and wf_doc["issuer"] not in self.keys._index:
            security["did_authenticity"] = False
            security["issues"].append(_issue("workflow_did_resolution_failed", "critical", wf["workflow_vc_id"], "Failed to resolve workflow VC issuer DID"))
        elif not verdict:
            security["key_validation"] = False
            security["issues"].append(_issue("workflow_signature_verification_failed", "critical", wf["workflow_vc_id"],
                                             "Workflow VC signature verification failed"))
        if not {"VerifiableCredential", "AgentFieldWorkflowCredential"} <= set(wf_doc.get("type") or []):
            compliance["agentfield_standard_compliance"] = False
            compliance["issues"].append(_issue("workflow_compliance_failure", "warning", wf["workflow_vc_id"],
                                               "Workflow VC does not meet AgentField standard requirements"))

    def verify_execution_vc_comprehensive(self, record, verification_timestamp=""):
        """VerifyExecutionVCComprehensive (vc_service.go:926-1005) of one ExecutionVC record (the dict vc_store.ExecutionVCStore returns,
        vc_document as str or bytes).  The caller passes the record, so the vc_not_found / system_disabled branches do not arise; a
        document that does not parse gives the early result (parse_error, score 0).  The signature goes through _keyed_verify."""
        try:
            doc = _parse_execution_doc(record["vc_document"])
        except (ValueError, KeyError, TypeError) as ex:
            return _parse_error_result(record, ex, verification_timestamp)
        verdict = self._keyed_verify([doc["issuer"]], [go_json.vc_document(doc)], [doc["proof"]["proofValue"]])[0]
        integrity, security, compliance = _new_checks()
        self._audit_component(record, doc, verdict, integrity, security, compliance)
        return _comprehensive_result([], integrity, security, compliance, verification_timestamp)

    def verify_workflow_vc_comprehensive(self, chain):
        """VerifyWorkflowVCComprehensive (vc_service.go:1386-1586) over one workflow's VC chain: chain = {"component_vcs": [ExecutionVC
        records: vc_id, execution_id, workflow_id, session_id, issuer_did, target_did, caller_did, vc_document (bytes), signature,
        input_hash, output_hash, status], "workflow_vc": WorkflowVC record or None}.  Every signature of the chain — the component
        VCs' and the workflow VC's — goes through ONE keyed GPU batch (the reference verifies them one by one, :1442-1546).
        `verification_timestamp` is the caller's (the reference reads the clock)."""
        integrity, security, compliance = _new_checks()
        critical = []
        parsed = []
        for ev in chain["component_vcs"]:
            try:
                parsed.append((ev, _parse_execution_doc(ev["vc_document"])))
            except (ValueError, KeyError, TypeError) as ex:
                critical.append(_issue("parse_error", "critical", ev["vc_id"], "Failed to parse VC document: %s" % ex))
        wf, wf_doc = chain.get("workflow_vc"), None
        if wf is not None and wf.get("vc_document") is not None:
            try:
                wf_doc = _parse_workflow_doc(wf["vc_document"])
            except (ValueError, KeyError, TypeError) as ex:
                critical.append(_issue("workflow_vc_parse_error", "critical", wf["workflow_vc_id"], "Failed to parse workflow VC document: %s" % ex))
        # one GPU batch for every signature of the chain
        dids = [d["issuer"] for _, d in parsed] + ([wf_doc["issuer"]] if wf_doc else [])
        msgs = [go_json.vc_document(d) for _, d in parsed] + ([go_json.workflow_vc_document(wf_doc)] if wf_doc else [])
        pvs = [d["proof"]["proofValue"] for _, d in parsed] + ([wf_doc["proof"]["proofValue"]] if wf_doc else [])
        verdicts = self._keyed_verify(dids, msgs, pvs) if dids else []
        for (ev, doc), verdict in zip(parsed, verdicts):
            self._audit_component(ev, doc, verdict, integrity, security, compliance)
        if wf_doc is not None:
            self._audit_workflow_vc(wf, wf_doc, verdicts[-1], security, compliance)
        return _comprehensive_result(critical, integrity, security, compliance, chain.get("verification_timestamp", ""))

    # -- the comprehensive audit on the device (afc_vc_audit_stored_batch)
    def _audit_device(self, kind, docs, columns):
        """(status, issue mask) per stored document from the device, or all HOST when there is no key set to resolve against."""
        n = len(docs)
        ks = self._named_keyset()
        if ks is None or not n:
            return np.full(n, _abi.VC_HOST, dtype=np.uint8), np.zeros(n, dtype=np.uint32)
        return ks.audit_stored(kind, docs, columns)

    def _host_verdicts(self, kind, parsed):
        """_keyed_verify over (index, parsed document) pairs the device left to the host: the mirror's own re-marshal and verify."""
        if not parsed:
            return {}
        marshal = go_json.vc_document if kind == _abi.DOC_EXECUTION_VC else go_json.workflow_vc_document
        v = self._keyed_verify([d["issuer"] for _, d in parsed], [marshal(d) for _, d in parsed], [d["proof"]["proofValue"] for _, d in parsed])
        return {i: x for (i, _), x in zip(parsed, v)}

    def audit_stored_execution_vcs(self, records, verification_timestamp=""):
        """verify_execution_vc_comprehensive for many ExecutionVC records (e.g. a whole store), one result per record and equal to it.
        One device call proves each stored document canonical, compares it with the record's columns, applies the timestamp,
        structure and compliance rules and verifies its signature.  A credential with nothing to report (verified, mask 0) gets the
        clean result without being parsed here; only documents the device left to the host (HOST), non-zero masks and undecided
        rules go through the mirror's checks, with the device's signature verdict where it has one."""
        docs = [_doc_bytes(r["vc_document"]) for r in records]
        status, issues = self._audit_device(_abi.DOC_EXECUTION_VC, docs, [[r[c] for c in _abi.AUDIT_COLUMNS] for r in records])
        out = [None] * len(records)
        host, report = [], []
        for i, (st, m) in enumerate(zip(status, issues)):
            if st == _abi.VC_VALID and m == 0:
                out[i] = _clean_result(verification_timestamp)
                continue
            try:
                doc = _parse_execution_doc(records[i]["vc_document"])
            except (ValueError, KeyError, TypeError) as ex:
                out[i] = _parse_error_result(records[i], ex, verification_timestamp)
                continue
            (host if st == _abi.VC_HOST else report).append((i, doc))
        verdicts = self._host_verdicts(_abi.DOC_EXECUTION_VC, host)
        for i, doc in host + report:
            verdict = verdicts[i] if i in verdicts else _device_verdict(status[i])
            integrity, security, compliance = _new_checks()
            self._audit_component(records[i], doc, verdict, integrity, security, compliance)
            out[i] = _comprehensive_result([], integrity, security, compliance, verification_timestamp)
        return out

    def audit_workflow_chains(self, chains):
        """verify_workflow_vc_comprehensive for many chains (same results, same issue order, same scores): the component documents
        of all chains go through one device call, the workflow VCs through a second.  Components and workflow VCs with nothing to
        report contribute nothing; the others go through the mirror's checks as in audit_stored_execution_vcs."""
        comps = [(c, ev) for c, ch in enumerate(chains) for ev in ch["component_vcs"]]
        c_status, c_issues = self._audit_device(_abi.DOC_EXECUTION_VC, [_doc_bytes(ev["vc_document"]) for _, ev in comps],
                                                [[ev[k] for k in _abi.AUDIT_COLUMNS] for _, ev in comps])
        wfs = [(c, ch["workflow_vc"]) for c, ch in enumerate(chains) if ch.get("workflow_vc") is not None and ch["workflow_vc"].get("vc_document") is not None]
        w_status, w_issues = self._audit_device(_abi.DOC_WORKFLOW_VC, [_doc_bytes(wf["vc_document"]) for _, wf in wfs], None)
        per_chain = [{"critical": [], "comps": [], "wf": None} for _ in chains]
        host_c, host_w = [], []
        for j, ((c, ev), st, m) in enumerate(zip(comps, c_status, c_issues)):
            if st == _abi.VC_VALID and m == 0:
                continue
            try:
                doc = _parse_execution_doc(ev["vc_document"])
            except (ValueError, KeyError, TypeError) as ex:
                per_chain[c]["critical"].append(_issue("parse_error", "critical", ev["vc_id"], "Failed to parse VC document: %s" % ex))
                continue
            per_chain[c]["comps"].append((j, ev, doc))
            if st == _abi.VC_HOST:
                host_c.append((j, doc))
        for j, ((c, wf), st, m) in enumerate(zip(wfs, w_status, w_issues)):
            if st == _abi.VC_VALID and m == 0:
                continue
            try:
                wf_doc = _parse_workflow_doc(wf["vc_document"])
            except (ValueError, KeyError, TypeError) as ex:
                per_chain[c]["critical"].append(_issue("workflow_vc_parse_error", "critical", wf["workflow_vc_id"],
                                                       "Failed to parse workflow VC document: %s" % ex))
                continue
            per_chain[c]["wf"] = (j, wf, wf_doc)
            if st == _abi.VC_HOST:
                host_w.append((j, wf_doc))
        c_verdicts = self._host_verdicts(_abi.DOC_EXECUTION_VC, host_c)
        w_verdicts = self._host_verdicts(_abi.DOC_WORKFLOW_VC, host_w)
        out = []
        for ch, p in zip(chains, per_chain):
            integrity, security, compliance = _new_checks()
            for j, ev, doc in p["comps"]:
                self._audit_component(ev, doc, c_verdicts[j] if j in c_verdicts else _device_verdict(c_status[j]), integrity, security, compliance)
            if p["wf"] is not None:
                j, wf, wf_doc = p["wf"]
                self._audit_workflow_vc(wf, wf_doc, w_verdicts[j] if j in w_verdicts else _device_verdict(w_status[j]), security, compliance)
            out.append(_comprehensive_result(p["critical"], integrity, security, compliance, ch.get("verification_timestamp", "")))
        return out


def _marshal_time(t) -> str:
    """Time.MarshalJSON of an aware datetime (microsecond precision): RFC3339Nano, Z for a zero offset."""
    off = int(t.utcoffset().total_seconds())
    text = "%04d-%02d-%02dT%02d:%02d:%02d" % (t.year, t.month, t.day, t.hour, t.minute, t.second)
    if t.microsecond:
        text += ("." + "%06d" % t.microsecond).rstrip("0")
    if off == 0:
        return text + "Z"
    a = abs(off) // 60
    return text + "%s%02d:%02d" % ("-" if off < 0 else "+", a // 60, a % 60)


def _compact(raw: bytes) -> bytes:
    """appendCompact(dst, raw, escapeHTML=true), which json.Marshal runs over a RawMessage; ValueError where it fails."""
    if not raw:
        raise ValueError("json: error calling MarshalJSON for type json.RawMessage: unexpected end of JSON input")
    json.loads(raw.decode("utf-8", "surrogateescape"), parse_constant=_reject_constant)
    out, in_str, esc, i = bytearray(), False, False, 0
    while i < len(raw):
        c = raw[i]
        if c in b"<>&":
            out += b"\\u00%02x" % c
        elif c == 0xE2 and raw[i + 1:i + 3] in (b"\x80\xa8", b"\x80\xa9") and i + 2 < len(raw):
            out += b"\\u202" + (b"8" if raw[i + 2] == 0xA8 else b"9")
            i += 3
            continue
        elif in_str:
            out.append(c)
            esc, in_str = (False, in_str) if esc else (c == 0x5C, c != 0x22)
        elif c not in b" \t\n\r":
            out.append(c)
            in_str = c == 0x22
        i += 1
    return bytes(out)


def _reject_constant(name):
    raise ValueError("invalid character %r" % name)


def workflow_chain_body(w, wvc, keys) -> bytes:
    """json.Marshal(types.WorkflowVCChainResponse) for one workflow on the host: w as get_workflow_vc_chain_batch takes it, wvc its
    issue_workflow_vc_batch result, keys the registry's public keys by DID (bytes)."""
    S = go_json.any_string
    evs = w["execution_vcs"]
    recs = []
    for v in evs:
        parts = ['"vc_id":' + S(v["vc_id"]), '"execution_id":' + S(v["execution_id"]), '"workflow_id":' + S(v["workflow_id"]),
                 '"session_id":' + S(v["session_id"])]
        for k in ("agent_node_id", "workflow_name"):
            if v.get(k) is not None:
                parts.append('"%s":' % k + S(v[k]))
        doc = "null" if v.get("vc_document") is None else _compact(bytes(v["vc_document"])).decode("utf-8", "surrogateescape")
        parts += ['"issuer_did":' + S(v["issuer_did"]), '"target_did":' + S(v["target_did"]), '"caller_did":' + S(v["caller_did"]),
                  '"vc_document":' + doc, '"signature":' + S(v["signature"]), '"storage_uri":' + S(v["storage_uri"]),
                  '"document_size_bytes":%d' % v["document_size_bytes"], '"input_hash":' + S(v["input_hash"]), '"output_hash":' + S(v["output_hash"]),
                  '"status":' + S(v["status"]), '"created_at":"%s"' % _marshal_time(v["created_at"])]
        recs.append("{" + ",".join(parts) + "}")
    times = [v["created_at"] for v in evs]
    start = min(times) if evs else w["snapshot"]
    wf = ['"workflow_id":' + S(w["workflow_id"]), '"session_id":' + S(wvc["session_id"]), '"component_vcs":' + "[" + ",".join(S(x) for x in wvc["component_vcs"]) + "]",
          '"workflow_vc_id":' + S(w["workflow_vc_id"]), '"status":' + S(wvc["status"]), '"start_time":"%s"' % _marshal_time(evs[times.index(start)]["created_at"] if evs else start)]
    if wvc["end_time"] is not None:
        wf.append('"end_time":"%s"' % _marshal_time(evs[times.index(max(times))]["created_at"]))
    doc = wvc["vc_document"]
    wf += ['"total_steps":%d' % len(evs), '"completed_steps":%d' % wvc["completed_steps"], '"vc_document":' + doc.decode("utf-8", "surrogateescape")]
    if wvc["signature"]:
        wf.append('"signature":' + S(wvc["signature"]))
    if wvc["issuer_did"]:
        wf.append('"issuer_did":' + S(wvc["issuer_did"]))
    wf += ['"snapshot_time":"%s"' % _marshal_time(w["snapshot"]), '"storage_uri":""', '"document_size_bytes":%d' % len(doc)]
    top = ['"workflow_id":' + S(w["workflow_id"]), '"component_vcs":[' + ",".join(recs) + "]", '"workflow_vc":{' + ",".join(wf) + "}",
           '"total_steps":%d' % len(evs), '"status":' + S(wvc["status"])]
    enc = lambda x: x.encode("utf-8", "surrogatepass") if isinstance(x, str) else bytes(x)
    wanted = set()
    for d in [x for v in evs for x in (v["issuer_did"], v["caller_did"], v["target_did"])] + [wvc["issuer_did"]]:
        d = enc(d)
        if d in (b"", b"did:key:") or not d.decode("utf-8", "replace").strip(_GO_SPACE) or d not in keys:
            continue
        wanted.add(d)
    if wanted:
        ents = []
        for d in sorted(wanted):
            method = d.split(b":")[1] if len(d) > 4 and d[:4] == b"did:" else b"key"
            x = base64.urlsafe_b64encode(keys[d]).rstrip(b"=").decode()
            ents.append(S(d) + ':{"method":' + S(method) + ',"public_key_jwk":{"alg":"EdDSA","crv":"Ed25519","kty":"OKP","use":"sig","x":"' + x +
                        '"},"resolved_from":"bundled","resolved_at":' + S(w["resolved_at"]) + "}")
        top.append('"did_resolution_bundle":{' + ",".join(ents) + "}")
    return ("{" + ",".join(top) + "}").encode("utf-8", "surrogateescape")


_DID_COMPONENT_TYPES = ("agentfield_server", "agent", "reasoner", "skill")     # by _abi.DID_KIND_*


def _did_bytes(v):
    return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)


def resolve_body(did, identity):
    """GET /api/v1/did/resolve/:did on the host (did_handlers.go:73-94): (HTTP status, body).  identity: what ResolveDID returns for did —
    {"kind" (_abi.DID_KIND_*), "derivation_path", "function_name", "public_key_jwk"} — or None when it finds nothing."""
    S = lambda v: go_json.string_bytes(_did_bytes(v))
    did = _did_bytes(did)
    if not did:
        return 400, b'{"error":"DID parameter is required"}'
    if identity is None:
        return 404, b'{"error":"DID not found"}'
    body = ('{"component_type":"%s","derivation_path":%s,"did":%s,"function_name":%s,"public_key_jwk":%s}'
            % (_DID_COMPONENT_TYPES[identity["kind"]], S(identity["derivation_path"]), S(did), S(identity["function_name"]),
               S(identity["public_key_jwk"])))
    return 200, body.encode()


def _go_unmarshal_jwk(raw: bytes):
    """json.Unmarshal(raw, &map[string]interface{}): the value (a dict, or None for null), or ValueError with Go's message for a value of
    another type and for truncated text; other syntax errors carry Python's wording."""
    v = go_json.decode_execution_payload(raw) if raw.strip(b" \t\r\n") else raw
    if isinstance(v, (bytes, bytearray)):                       # rejected: a syntax error, or a number outside float64's range
        try:
            json.loads(go_json.go_utf8(raw))
        except ValueError as ex:
            if getattr(ex, "pos", 0) >= len(raw.rstrip(b" \t\r\n")):
                raise ValueError("unexpected end of JSON input")
            raise ValueError(str(ex))
        raise ValueError("json: cannot unmarshal number into Go value of type float64")
    if v is None or isinstance(v, dict):
        return v
    kind = "array" if isinstance(v, list) else "string" if isinstance(v, str) else "bool" if isinstance(v, bool) else "number"
    raise ValueError("json: cannot unmarshal %s into Go value of type map[string]interface {}" % kind)


def document_body(did, identity):
    """GET /api/v1/did/document/:did on the host (did_handlers.go:368-429): (HTTP status, body), identity as for resolve_body.  The stored
    JWK goes through json.Unmarshal into map[string]interface{} and back; a text Go rejects is a 500."""
    S = lambda v: go_json.string_bytes(_did_bytes(v))
    did = _did_bytes(did)
    if not did:
        return 400, b'{"error":"DID parameter is required"}'
    if identity is None:
        return 404, ('{"details":%s,"error":"DID not found"}' % S(b"DID not found: " + did)).encode()
    try:
        jwk = _go_unmarshal_jwk(_did_bytes(identity["public_key_jwk"]))
    except ValueError as ex:
        return 500, ('{"details":%s,"error":"Failed to parse public key"}' % S(str(ex))).encode()
    d, key = S(did), S(did + b"#key-1")
    body = ('{"@context":["https://www.w3.org/ns/did/v1","https://w3id.org/security/suites/ed25519-2020/v1"],"assertionMethod":[%s],'
            '"authentication":[%s],"id":%s,"service":[{"description":"AgentField Agent Platform Service","id":%s,'
            '"serviceEndpoint":"https://agentfield.example.com/api/v1","type":"AgentFieldAgentService"}],"verificationMethod":[{"controller":%s,'
            '"id":%s,"publicKeyJwk":%s,"type":"Ed25519VerificationKey2020"}]}'
            % (key, key, d, S(did + b"#agentfield-service"), d, key, go_json.value(jwk)))
    return 200, body.encode("utf-8", "surrogatepass")


_GO_SPACE ="\t\n\v\f\r \x85\xa0\u1680\u2000\u2001\u2002\u2003\u2004\u2005\u2006\u2007\u2008\u2009\u200a\u2028\u2029\u202f\u205f\u3000"


def _issue(kind, severity, component, description, field="", expected="", actual=""):
    """types.VerificationIssue (vc_service.go:880-889)."""
    return {"type": kind, "severity": severity, "component": component, "field": field, "expected": expected, "actual": actual,
            "description": description}


def _doc_bytes(doc):
    return doc.encode("utf-8") if isinstance(doc, str) else bytes(doc)


def _parse_execution_doc(raw):
    """What the comprehensive checks read a stored execution VC as (json.Unmarshal into types.VCDocument, numbers as float64)."""
    doc = json.loads(raw, parse_int=float)
    doc["credentialSubject"]["audit"]["metadata"] = go_json.unmarshal_numbers(doc["credentialSubject"]["audit"].get("metadata"))
    doc["credentialSubject"]["execution"].setdefault("errorMessage", "")
    return doc


def _parse_workflow_doc(raw):
    doc = json.loads(raw, parse_int=float)
    doc["credentialSubject"]["audit"]["metadata"] = go_json.unmarshal_numbers(doc["credentialSubject"]["audit"].get("metadata"))
    return doc


def _new_checks():
    """The three running results as performIntegrityChecks / performSecurityAnalysis / performComplianceChecks start them."""
    integrity = {"metadata_consistency": True, "field_consistency": True, "timestamp_validation": True, "hash_validation": True,
                 "structural_integrity": True, "issues": []}
    security = {"signature_strength": "Ed25519", "key_validation": True, "did_authenticity": True, "replay_protection": True,
                "tamper_evidence": [], "security_score": 100.0, "issues": []}
    compliance = {"w3c_compliance": True, "agentfield_standard_compliance": True, "audit_trail_integrity": True,
                  "data_integrity_checks": True, "issues": []}
    return integrity, security, compliance


def _comprehensive_result(critical, integrity, security, compliance, verification_timestamp):
    """ComprehensiveVCVerificationResult: issues split by severity, calculateOverallScore (vc_service.go:1361-1383)."""
    all_issues = integrity["issues"] + security["issues"] + compliance["issues"]
    critical = critical + [i for i in all_issues if i["severity"] == "critical"]
    warnings = [i for i in all_issues if i["severity"] == "warning"]
    score = max(0.0, ((100.0 - 25.0 * len(critical) - 5.0 * len(warnings)) + security["security_score"]) / 2.0)
    return {"valid": not critical, "overall_score": score, "critical_issues": critical, "warnings": warnings, "integrity_checks": integrity,
            "security_analysis": security, "compliance_checks": compliance, "verification_timestamp": verification_timestamp}


def _clean_result(verification_timestamp):
    """The result of a credential with nothing to report."""
    return _comprehensive_result([], *_new_checks(), verification_timestamp)


def _parse_error_result(record, ex, verification_timestamp):
    """VerifyExecutionVCComprehensive's early return when json.Unmarshal fails (vc_service.go:966-977): the three checks keep Go's zero values."""
    return {"valid": False, "overall_score": 0.0,
            "critical_issues": [_issue("parse_error", "critical", record["vc_id"], "Failed to parse VC document: %s" % ex)], "warnings": [],
            "integrity_checks": {"metadata_consistency": False, "field_consistency": False, "timestamp_validation": False, "hash_validation": False,
                                 "structural_integrity": False, "issues": None},
            "security_analysis": {"signature_strength": "", "key_validation": False, "did_authenticity": False, "replay_protection": False,
                                  "tamper_evidence": None, "security_score": 0.0, "issues": None},
            "compliance_checks": {"w3c_compliance": False, "agentfield_standard_compliance": False, "audit_trail_integrity": False,
                                  "data_integrity_checks": False, "issues": None},
            "verification_timestamp": verification_timestamp}


def _device_verdict(status):
    """A device status as _keyed_verify's verdict: VALID True, INVALID False, UNRESOLVED / BAD_ENCODING None."""
    return {_abi.VC_VALID: True, _abi.VC_INVALID: False}.get(int(status))


def _vc_response(valid, error="", message="", issuer_did="", issued_at=""):
    """types.VCVerificationResponse (pkg/types/did_types.go:273-279); "" stands for an omitted field."""
    return {"valid": valid, "error": error, "message": message, "issuer_did": issuer_did, "issued_at": issued_at}


def _b64url_error_at(s: str) -> int:
    """The input byte base64.RawURLEncoding.DecodeString reports in its CorruptInputError: the first character outside the URL
    alphabet, else (length = 1 mod 4) the last one."""
    import re
    m = re.search(r"[^A-Za-z0-9_-]", s)
    return m.start() if m else len(s) - 1


def _response_bytes(r) -> bytes:
    """json.Marshal(types.VCVerificationResponse) of a _vc_response dict: field order, omitempty, Go's escaping."""
    out = '{"valid":%s' % ("true" if r["valid"] else "false")
    for key, name in (("issuer_did", "issuer_did"), ("issued_at", "issued_at"), ("message", "message"), ("error", "error")):
        if r[key]:
            out += ',"%s":%s' % (name, go_json.string(r[key]))
    return (out + "}").encode("utf-8", "surrogatepass")


_ABSENT = object()


def _go_fold(name: str) -> str:
    """encoding/json's foldName: ASCII letters upper-cased, every other rune mapped through ToUpper(ToLower(r))."""
    out = []
    for ch in name:
        if ch < "\x80":
            out.append(ch.upper() if "a" <= ch <= "z" else ch)
        else:
            f = ch.lower()
            f = f.upper() if len(f) == 1 else ch
            out.append(f if len(f) == 1 else ch)
    return "".join(out)


def _bind_verify_request(raw: bytes):
    """c.ShouldBindJSON(&types.VCVerificationRequest) with gin's default decoder: the first JSON value of the body (what follows it is not
    read), which must be an object or null.  Returns the decoded vc_document value (the last member whose name matches it exactly or
    folded), _ABSENT when there is none; raises ValueError where the bind fails."""
    text = raw.decode("utf-8", "surrogateescape")
    i = 0
    while i < len(text) and text[i] in " \t\n\r":
        i += 1

    def no_constants(name):
        raise ValueError("invalid character in numeric literal: %s" % name)
    try:
        v, _ = json.JSONDecoder(object_pairs_hook=_Obj, parse_constant=no_constants).raw_decode(text, i)
    except ValueError:
        raise ValueError("invalid request body")
    if v is None:
        return _ABSENT
    if not isinstance(v, _Obj):
        raise ValueError("json: cannot unmarshal into Go value of type types.VCVerificationRequest")
    want = _go_fold("vc_document")
    found = _ABSENT
    for k, x in v:
        if k == "vc_document" or _go_fold(k) == want:
            found = x
    return found


class _Obj(list):
    """A JSON object as its (key, value) pairs in document order (json.loads object_pairs_hook)."""


_STR, _STRLIST, _INT, _PTRSTR, _MAP = "string", "[]string", "int", "*string", "map[string]interface {}"
_CALLER = {"did": _STR, "type": _STR, "agentNodeDid": _STR}
_AUDIT = {"inputDataHash": _STR, "outputDataHash": _STR, "metadata": _MAP}
_PROOF = {"type": _STR, "created": _STR, "verificationMethod": _STR, "proofPurpose": _STR, "proofValue": _STR}
_VC_DOC = {"@context": _STRLIST, "type": _STRLIST, "id": _STR, "issuer": _STR, "issuanceDate": _STR,
           "credentialSubject": {"executionId": _STR, "workflowId": _STR, "sessionId": _STR, "caller": _CALLER,
                                 "target": {"did": _STR, "agentNodeDid": _STR, "functionName": _STR},
                                 "execution": {"inputHash": _STR, "outputHash": _STR, "timestamp": _STR, "durationMs": _INT, "status": _STR,
                                               "errorMessage": _STR},
                                 "audit": _AUDIT},
           "proof": _PROOF}
_WF_DOC = {"@context": _STRLIST, "type": _STRLIST, "id": _STR, "issuer": _STR, "issuanceDate": _STR,
           "credentialSubject": {"workflowId": _STR, "sessionId": _STR, "componentVcIds": _STRLIST, "totalSteps": _INT, "completedSteps": _INT,
                                 "status": _STR, "startTime": _STR, "endTime": _PTRSTR, "snapshotTime": _STR, "orchestrator": _CALLER,
                                 "audit": _AUDIT},
           "proof": _PROOF}


def _zero(t):
    if isinstance(t, dict):
        return {k: _zero(v) for k, v in t.items()}
    return {_STR: "", _INT: 0}.get(t)


def _interface(v):
    """json.Unmarshal into interface{}: objects -> maps (the last duplicate wins), numbers -> float64."""
    if isinstance(v, _Obj):
        return {k: _interface(x) for k, x in v}
    if isinstance(v, list):
        return [_interface(x) for x in v]
    return go_json.unmarshal_numbers(v)


def _go_into(v, t, cur):
    """Decodes JSON value v into a Go value of type t whose current value is cur (json.Unmarshal: null leaves non-pointer values
    alone, struct members match exactly or else case-insensitively, unknown members are ignored)."""
    if isinstance(t, dict):
        if v is None:
            return cur
        if not isinstance(v, _Obj):
            raise ValueError("json: cannot unmarshal into Go struct")
        for k, x in v:
            name = k if k in t else next((f for f in t if f.lower() == k.lower()), None)
            if name is not None:
                cur[name] = _go_into(x, t[name], cur[name])
        return cur
    if t in (_STR, _PTRSTR):
        if v is None:
            return None if t == _PTRSTR else cur
        if not isinstance(v, str):
            raise ValueError("json: cannot unmarshal %s into Go value of type string" % type(v).__name__)
        return v
    if t == _STRLIST:
        if v is None:
            return None
        if not isinstance(v, list) or isinstance(v, _Obj) or not all(x is None or isinstance(x, str) for x in v):
            raise ValueError("json: cannot unmarshal into Go value of type []string")
        return ["" if x is None else x for x in v]
    if t == _INT:
        if v is None:
            return cur
        if isinstance(v, bool) or not isinstance(v, int) or not -2**63 <= v < 2**63:
            raise ValueError("json: cannot unmarshal number into Go value of type int")
        return v
    if v is None:                                   # map
        return None
    if not isinstance(v, _Obj):
        raise ValueError("json: cannot unmarshal into Go value of type map[string]interface {}")
    return _interface(v)


def go_unmarshal_vc(raw: bytes, kind=0):
    """json.Unmarshal(raw, &types.VCDocument) (kind 0) or &types.WorkflowVCDocument (kind 1) as the host mirror's dict; raises
    ValueError where Go returns an error."""
    import json
    try:
        v = json.loads(raw.decode("utf-8", "replace"), object_pairs_hook=_Obj)
    except ValueError as ex:
        raise ValueError(str(ex))
    schema = _VC_DOC if kind == 0 else _WF_DOC
    return _go_into(v, schema, _zero(schema))


def _b64url_decode_strict(s: str) -> bytes:
    """base64.RawURLEncoding.DecodeString: URL alphabet, no padding, no stray characters (Go returns an error otherwise)."""
    import re
    if not re.fullmatch(r"[A-Za-z0-9_-]*", s) or len(s) % 4 == 1:
        raise ValueError("illegal base64 data")
    raw = base64.urlsafe_b64decode(s + "=" * (-len(s) % 4))
    if _b64url(raw) != s:                      # non-zero trailing bits: Go's strict decoder accepts them, Python ignores them too
        pass
    return raw


def _is_rfc3339(ts: str) -> bool:
    """time.Parse(time.RFC3339, ts) == nil (vc_service.go:1248-1251), for the forms the control plane emits and the obvious
    malformed ones: date, 'T', time, optional fraction, 'Z' or a numeric offset."""
    import re
    m = re.fullmatch(r"(\d{4})-(\d{2})-(\d{2})T(\d{2}):(\d{2}):(\d{2})(\.\d+)?(Z|[+-](\d{2}):(\d{2}))", ts)
    if not m:
        return False
    mo, d, h, mi, sec = (int(m.group(i)) for i in (2, 3, 4, 5, 6))
    if not (1 <= mo <= 12 and 1 <= d <= 31 and h <= 23 and mi <= 59 and sec <= 59):
        return False
    if m.group(9) is not None and not (int(m.group(9)) <= 23 and int(m.group(10)) <= 59):
        return False
    import calendar
    return d <= calendar.monthrange(int(m.group(1)), mo)[1]


class DIDService:
    """The registration half of the reference's DIDService (control-plane/internal/services/did_service.go:186-365, 653-723) over one
    registry: its server id, master seed and agent nodes.  Every new agent's keys, DIDs and DIDRegistrationResponse come from one
    afc_did_register_batch call (ExpandedKeys.register), and the keys join `keys`, so the agents can issue credentials at once.  Known
    agents take RegisterAgent's other branch (:154-179: the differential analysis, DeregisterComponents, PartialRegisterAgent or the
    existing identity package) through one afc_did_reregister_batch call (ExpandedKeys.reregister); register_agents takes a mixed batch.
    The agent index of a known agent's new components is the <a> of its own stored path (the reference uses its place in Go's randomised
    map iteration)."""

    def __init__(self, keys: ExpandedKeys, master_seed: bytes, server_id):
        if len(master_seed) != 32:
            raise ValueError("the master seed is 32 bytes")
        self.keys = keys
        self.master_seed = bytes(master_seed)
        self.server_id = server_id.encode() if isinstance(server_id, str) else bytes(server_id)
        # node id (bytes) -> {"did", "derivation_path", "public_key_jwk", "reasoners": {id: component}, "skills": {id: component}}, a
        # component being {"did", "derivation_path", "public_key_jwk", "function_name"}: what the existing identity package needs
        self.agent_nodes = {}
        self._resolver = None             # serve_did_requests: (DIDDirectory with identities, DID bytes -> identity)

    @staticmethod
    def _node_key(v):
        return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)

    def _register(self, requests):
        self._resolver = None                                     # serve_did_requests rebuilds its directory
        results = self.keys.register(self.master_seed, self.server_id, requests, len(self.agent_nodes))
        for r, res in zip(requests, results):
            comps = res["components"]
            entry = {"did": comps[0]["did"], "derivation_path": comps[0]["path"], "public_key_jwk": public_jwk(comps[0]["pk"]), "reasoners": {},
                     "skills": {}}
            for c in comps[1:]:
                if c["kept"]:
                    k = self._node_key(c["id"])
                    entry["reasoners" if c["type"] == "reasoner" else "skills"][k] = {"did": c["did"], "derivation_path": c["path"],
                                                                                     "public_key_jwk": public_jwk(c["pk"]), "function_name": k}
            self.agent_nodes[self._node_key(r["agent_node_id"])] = entry
        return results

    def register_agents_batch(self, requests):
        """handleNewRegistration for new agents, in order (request k gets agent index len(registry) + k).  A node id already registered,
        or repeated in the batch, raises ValueError: a known node takes reregister_agents_batch or register_agents.  Returns per request {"body", "components"}."""
        seen = set()
        for r in requests:
            k = self._node_key(r["agent_node_id"])
            if k in self.agent_nodes or k in seen:
                raise ValueError("agent node %r is already registered" % k)
            seen.add(k)
        return self._register(requests)

    def backfill_existing_nodes(self, nodes):
        """BackfillExistingNodes: every node ({"agent_node_id", "reasoners", "skills"}) the registry lacks is registered, in list order,
        in one call; registered nodes (and later repeats of a node) are skipped.  Returns the new nodes' results."""
        todo, seen = [], set()
        for r in nodes:
            k = self._node_key(r["agent_node_id"])
            if k in self.agent_nodes or k in seen:
                continue
            seen.add(k)
            todo.append(r)
        return self._register(todo) if todo else []

    ROOT_PATH = "m/44'/0'"

    @property
    def root_did(self):
        """registry.RootDID: generateDIDFromSeed(masterSeed, "m/44'/0'") (did_service.go:61); its key joins `keys`, since the workflow
        credential of a workflow without records is issued under it (vc_service.go:577-580)."""
        if getattr(self, "_root_did", None) is None:
            self._root_did = self.keys.derive(self.master_seed, [self.ROOT_PATH])[0]
        return self._root_did

    def _identities(self):
        """Every DID ResolveDID resolves (did_service.go:368-473), each once, in registration order — the root DID, then each agent, its
        reasoners and its skills in insertion order — as DID -> {"pk", "kind", "derivation_path", "function_name", "public_key_jwk"}.  A DID
        the registry holds twice (re-registration gives every new component of one kind the same DID) keeps its first holder: Go's
        randomised map iteration may return any of them, and they differ only in function_name."""
        root_pk = self.keys.public_key(self.root_did)
        out = {self.root_did: {"pk": root_pk, "kind": _abi.DID_KIND_SERVER, "derivation_path": self.ROOT_PATH, "function_name": b"",
                               "public_key_jwk": public_jwk(root_pk)}}
        for a in self.agent_nodes.values():
            comps = [(a, _abi.DID_KIND_AGENT)] + [(c, _abi.DID_KIND_REASONER) for c in a["reasoners"].values()] + \
                    [(c, _abi.DID_KIND_SKILL) for c in a["skills"].values()]
            for e, kind in comps:
                if e["did"] not in out:
                    x = json.loads(e["public_key_jwk"])["x"]
                    out[e["did"]] = {"pk": base64.urlsafe_b64decode(x + "=" * (-len(x) % 4)), "kind": kind, "derivation_path": e["derivation_path"],
                                     "function_name": e.get("function_name", b""), "public_key_jwk": e["public_key_jwk"]}
        return out

    def did_directory(self, ctx=None, identities=False):
        """The registry's public half on the device (identity.DIDDirectory): every DID ResolveDID resolves with its public key — the root
        DID (the key at m/44'/0'), then every agent's and component's DID with the key its stored public JWK holds (the JWK's x), each
        once (_identities).  With `identities` the directory also holds what DID resolution and DID documents need (set_identities)."""
        return self._directory(self._identities(), ctx, identities)

    def _directory(self, ids, ctx=None, identities=False):
        from .identity import DIDDirectory
        d = DIDDirectory(list(ids), [e["pk"] for e in ids.values()], ctx=ctx or self.keys.ctx)
        if identities:
            d.set_identities(*[[e[k] for e in ids.values()] for k in ("kind", "derivation_path", "function_name", "public_key_jwk")])
        return d

    def serve_did_requests(self, requests):
        """GET /api/v1/did/resolve/:did and GET /api/v1/did/document/:did for many requests, [(kind, did)] with kind _abi.DIDRES_RESOLVE or
        _DOCUMENT, in one device call (identity.DIDDirectory.resolve) over a directory with identities, rebuilt after a registration.
        Returns [(HTTP status, body)] in request order; requests the device leaves to the host go through resolve_body / document_body."""
        for kind, _ in requests:
            if kind not in (_abi.DIDRES_RESOLVE, _abi.DIDRES_DOCUMENT):
                raise ValueError("unknown request kind %r" % kind)
        if self._resolver is None:
            ids = self._identities()
            self._resolver = (self._directory(ids, identities=True), {_did_bytes(k): v for k, v in ids.items()})
        directory, index = self._resolver
        status = {_abi.DIDRES_FOUND: 200, _abi.DIDRES_NOT_FOUND: 404, _abi.DIDRES_BAD_REQUEST: 400}
        out = []
        for (kind, did), (st, body) in zip(requests, directory.resolve(requests) if requests else []):
            if st == _abi.DIDRES_HOST:
                host = resolve_body if kind == _abi.DIDRES_RESOLVE else document_body
                out.append(host(did, index.get(_did_bytes(did))))
            else:
                out.append((status[st], body))
        return out

    def _reregister(self, requests):
        self._resolver = None
        reqs = []
        for r in requests:
            a = self.agent_nodes[self._node_key(r["agent_node_id"])]
            reqs.append({"agent": a, "reasoners": r.get("reasoners") or (), "skills": r.get("skills") or ()})
        results = self.keys.reregister(self.master_seed, self.server_id, reqs)
        for q, res in zip(reqs, results):                         # the registry update: GONE first, then the kept NEW ids
            a = q["agent"]
            for kind, name in ((0, "reasoners"), (1, "skills")):
                for key, gone in zip(list(a[name]), res["gone"][kind]):
                    if gone:
                        del a[name][key]
                slot = res["slots"][kind]
                for x in res["new"][kind]:
                    k = self._node_key(x)
                    a[name][k] = {"did": slot["did"], "derivation_path": slot["path"], "public_key_jwk": slot["public_key_jwk"], "function_name": k}
        return results

    def _distinct(self, requests):
        seen = set()
        for r in requests:
            k = self._node_key(r["agent_node_id"])
            if k in seen:
                raise ValueError("agent node %r is named twice in one batch" % k)
            seen.add(k)

    def reregister_agents_batch(self, requests):
        """RegisterAgent for agents the registry holds ({"agent_node_id", "reasoners", "skills"}): the removed components leave the registry
        and the new ones join it with their keys (which join `keys`).  An unknown node, or one named twice, raises ValueError.  Returns per
        request {"state", "counts", "body", "gone", "new", "slots"} (ExpandedKeys.reregister)."""
        self._distinct(requests)
        for r in requests:
            if self._node_key(r["agent_node_id"]) not in self.agent_nodes:
                raise ValueError("agent node %r is not registered" % self._node_key(r["agent_node_id"]))
        return self._reregister(requests) if requests else []

    def register_agents(self, requests):
        """RegisterAgent over a mixed batch: new nodes through one afc_did_register_batch call (request order gives their agent indices),
        known nodes through one afc_did_reregister_batch call.  A node named twice raises ValueError (the reference handles requests one
        after another, so a second request for a node would see the first one's result).  Returns the results in request order: those of
        register_agents_batch for new nodes, of reregister_agents_batch for known ones."""
        self._distinct(requests)
        known = [k for k, r in enumerate(requests) if self._node_key(r["agent_node_id"]) in self.agent_nodes]
        fresh = [k for k, r in enumerate(requests) if self._node_key(r["agent_node_id"]) not in self.agent_nodes]
        out = [None] * len(requests)
        if known:
            for k, res in zip(known, self._reregister([requests[k] for k in known])):
                out[k] = res
        if fresh:
            for k, res in zip(fresh, self._register([requests[k] for k in fresh])):
                out[k] = res
        return out
