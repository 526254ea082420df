"""Host-side mirror of the Go `internal/identity` package this build adds (SURVEY.md §8b, §8f N1): the key cache.

Two caches, both replacing work the reference redoes on every request:

  * ExpandedKeys — DID -> (clamped scalar s, prefix, pk) so that issuing a VC costs one fixed-base multiplication
    instead of the three the reference performs (NewKeyFromSeed inside every ResolveDID, did_service.go:515-525,585-599;
    NewKeyFromSeed again in signVC, vc_service.go:460; then Sign, :463).
  * KeySet — a set of issuer public keys with per-key radix-256 tables on the GPU, so that verification against a
    known issuer needs no doublings (VerifyVC resolves the issuer from the registry first, vc_service.go:259;
    VerifyWorkflowVCComprehensive loops over one workflow's VCs, :1442-1512).

Derivation follows the reference exactly: seed' = SHA-256(masterSeed || path), did:key = "did:key:z" + base64url(0xED 0x01 || pk)
(did_service.go:515-536 — base64url, not base58btc, despite the 'z').
"""
import base64
import ctypes as C
import datetime

import numpy as np

from . import _abi
from .crypto import default_context, pack


def did_key(pk: bytes) -> str:
    return "did:key:z" + base64.urlsafe_b64encode(b"\xed\x01" + pk).rstrip(b"=").decode()


class ExpandedKeys:
    """DID -> expanded signing key, filled in bulk on the GPU."""

    def __init__(self, ctx=None):
        self.ctx = ctx or default_context()
        self._index = {}
        self._expanded = np.zeros((0, 96), dtype=np.uint8)

    def derive(self, master_seed: bytes, paths):
        """derivePrivateKey for many paths at once: returns the DIDs, in order, and caches their expanded keys."""
        buf, off = pack([master_seed + p.encode() for p in paths])
        seeds = self.ctx.sha256_packed(buf, off)                 # SHA-256(masterSeed || path)
        exp = self.ctx.expand(seeds)
        dids = [did_key(bytes(e[64:])) for e in exp]
        base = self._expanded.shape[0]
        self._expanded = np.concatenate([self._expanded, exp])
        for i, d in enumerate(dids):
            self._index[d] = base + i
        return dids

    def public_key(self, did):
        return bytes(self._expanded[self._index[did], 64:])

    def sign_batch(self, dids, msgs):
        """signVC for a batch: one fixed-base multiplication per credential."""
        ki = np.fromiter((self._index[d] for d in dids), dtype=np.uint32, count=len(dids))
        buf, off = pack(msgs)
        return [bytes(s) for s in self.ctx.sign_expanded_packed(self._expanded, ki, buf, off)]

    def sign_dev(self, dids, d_msgs, d_off, n):
        """The same for messages already on the device (e.g. assembled there by canonical.JsonTemplate.fill_dev)."""
        import torch
        dev = d_off.device
        ki = np.fromiter((self._index[d] for d in dids), dtype=np.uint32, count=len(dids))
        d_exp = torch.from_numpy(self._expanded).to(dev)
        d_ki = torch.from_numpy(ki.view(np.int32)).to(dev)
        d_sigs = torch.empty((n, 64), dtype=torch.uint8, device=dev)
        self.ctx.sign_expanded_dev(d_exp, d_ki, d_msgs, d_off, n, d_sigs)
        torch.cuda.synchronize(dev)
        return [bytes(s) for s in d_sigs.cpu().numpy()]

    def key_index(self, dids):
        return np.fromiter((self._index[d] for d in dids), dtype=np.uint32, count=len(dids))

    def _issue_bound(self, n, col_bytes):
        """afc_vc_issue_bound for n requests of col_bytes column bytes in all (the bound is a sum over requests)."""
        lib = _abi.load()
        one = np.zeros(len(_abi.ISSUE_COLUMNS) + 1, dtype=np.uint64)
        fixed = lib.afc_vc_issue_bound(_abi.ptr(one), 1)
        one[-1] = col_bytes
        return lib.afc_vc_issue_bound(_abi.ptr(one), 1) + (n - 1) * fixed if n else 0

    def issue_dev(self, d_key_index, d_cols, d_col_off, d_duration, d_payloads, d_payload_off, d_payload_nil, n, hash_data=True, log=None,
                  stream=None, d_expanded=None):
        """afc_vc_issue_execution_batch_dev: n GenerateExecutionVC requests on the device.  d_key_index: int32 [n] into this cache (or
        into d_expanded, K x 96); d_cols / d_col_off: uint8 columns and int64 [n*14+1] absolute offsets (_abi.ISSUE_COLUMNS order);
        d_duration: int64 [n]; d_payloads / d_payload_off (int64 [2n+1]) / d_payload_nil (uint8 [2n]): input i then output i, read only
        with hash_data; log: an audit.Auditor that receives the stored documents.  Returns (d_docs uint8, d_doc_off int64 [n+1],
        d_hashes uint8 [n, 86] or None, d_proof_values uint8 [n, 86])."""
        import torch
        dev = d_col_off.device
        if d_expanded is None:
            d_expanded = torch.from_numpy(self._expanded).to(dev)
        ncols = len(_abi.ISSUE_COLUMNS)
        col_bytes = int(d_col_off[n * ncols]) - int(d_col_off[0]) if n else 0
        cap = self._issue_bound(n, col_bytes)
        d_docs = torch.empty(max(cap, 1), dtype=torch.uint8, device=dev)
        d_doc_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_hashes = torch.empty((n, 86), dtype=torch.uint8, device=dev) if hash_data else None
        d_pv = torch.empty((n, 86), dtype=torch.uint8, device=dev)
        lib = _abi.load()
        _abi.check(lib.afc_vc_issue_execution_batch_dev(self.ctx.handle, _abi.ptr(d_expanded), d_expanded.shape[0], _abi.ptr(d_key_index),
                                                        _abi.ptr(d_cols), _abi.ptr(d_col_off), _abi.ptr(d_duration), _abi.ptr(d_payloads),
                                                        _abi.ptr(d_payload_off), _abi.ptr(d_payload_nil), _abi.ISSUE_HASH_DATA if hash_data else 0, n,
                                                        log.handle if log is not None else None, _abi.ptr(d_docs), cap, _abi.ptr(d_doc_off),
                                                        _abi.ptr(d_hashes), _abi.ptr(d_pv), self.ctx._stream(stream)), self.ctx.handle)
        total = int(d_doc_off[n]) if n else 0
        return d_docs[:total], d_doc_off, d_hashes, d_pv

    def issue_packed(self, key_index, cols, col_off, duration, payloads, payload_off, payload_nil, hash_data=True, log=None, expanded=None):
        """afc_vc_issue_execution_batch on host arrays (the layout of issue_dev).  Returns (docs uint8, doc_off uint64 [n+1], hashes
        uint8 [n, 86] or None, proof_values uint8 [n, 86])."""
        n = len(key_index)
        exp = self._expanded if expanded is None else expanded
        cap = _abi.load().afc_vc_issue_bound(_abi.ptr(col_off), n)
        docs = np.empty(max(cap, 1), dtype=np.uint8)
        doc_off = np.zeros(n + 1, dtype=np.uint64)
        hashes = np.empty((n, 86), dtype=np.uint8) if hash_data else None
        pv = np.empty((n, 86), dtype=np.uint8)
        _abi.check(_abi.load().afc_vc_issue_execution_batch(self.ctx.handle, _abi.ptr(exp), exp.shape[0], _abi.ptr(key_index), _abi.ptr(cols),
                                                            _abi.ptr(col_off), _abi.ptr(duration), _abi.ptr(payloads), _abi.ptr(payload_off),
                                                            _abi.ptr(payload_nil), _abi.ISSUE_HASH_DATA if hash_data else 0, n,
                                                            log.handle if log is not None else None, _abi.ptr(docs), cap, _abi.ptr(doc_off),
                                                            _abi.ptr(hashes), _abi.ptr(pv)), self.ctx.handle)
        return docs[:int(doc_off[n])], doc_off, hashes, pv

    @staticmethod
    def pack_issue_requests(requests):
        """GenerateExecutionVC requests (the dicts of services.VCService.generate_execution_vc_batch) -> (cols, col_off, duration, payloads,
        payload_off, payload_nil) host arrays.  Strings are UTF-8 with lone surrogates kept as their three bytes; bytes pass as they are."""
        defaults = {"caller_type": "agent", "target_did": "", "function_name": "", "error_message": ""}

        def col(r, k):
            v = r.get(k) if k in defaults else r[k]
            v = defaults[k] if v is None else v
            return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)
        flat = [col(r, k) for r in requests for k in _abi.ISSUE_COLUMNS]
        cols, col_off = pack(flat)
        duration = np.fromiter((int(r["duration_ms"]) for r in requests), dtype=np.int64, count=len(requests))
        pl = [(r.get("input"), r.get("output")) for r in requests]
        payloads, payload_off = pack([b"" if p is None else p for io in pl for p in io])
        payload_nil = np.fromiter((p is None for io in pl for p in io), dtype=np.uint8, count=2 * len(requests))
        return cols, col_off, duration, payloads, payload_off, payload_nil

    def issue(self, requests, hash_data=True, log=None):
        """GenerateExecutionVC for many requests in one host-buffer call: [{"vc_document": bytes, "signature": str, "input_hash": str,
        "output_hash": str}]."""
        n = len(requests)
        if n == 0:
            return []
        ki = self.key_index([r["caller_did"] for r in requests])
        docs, off, hashes, pv = self.issue_packed(ki, *self.pack_issue_requests(requests), hash_data=hash_data, log=log)
        buf = docs.tobytes()
        out = []
        for i in range(n):
            ih, oh = (hashes[i, :43].tobytes().decode(), hashes[i, 43:].tobytes().decode()) if hash_data else ("", "")
            out.append({"vc_document": buf[int(off[i]):int(off[i + 1])], "signature": pv[i].tobytes().decode(), "input_hash": ih, "output_hash": oh})
        return out

    # -- workflow credentials (afc_vc_issue_workflow_batch)
    _wf_coef = None

    @classmethod
    def _workflow_bound(cls, n, col_bytes, records, rec_bytes):
        """afc_vc_workflow_bound for n workflows with these totals, without building their offset arrays: the bound is linear in the four,
        so its coefficients are read off the library once."""
        if cls._wf_coef is None:
            lib = _abi.load()
            col_off = np.zeros(len(_abi.WORKFLOW_COLUMNS) + 1, dtype=np.uint64)
            rec_off = np.zeros(2, dtype=np.uint64)
            rec_col_off = np.zeros(3, dtype=np.uint64)

            def f():
                return lib.afc_vc_workflow_bound(_abi.ptr(col_off), _abi.ptr(rec_off), _abi.ptr(rec_col_off), 1)
            fixed = f()
            col_off[-1] = 1
            per_col = f() - fixed
            col_off[-1] = 0
            rec_off[1] = 1
            per_rec = f() - fixed
            rec_col_off[2] = 1
            per_rec_byte = f() - fixed - per_rec
            cls._wf_coef = (fixed, per_col, per_rec, per_rec_byte)
        fixed, per_col, per_rec, per_rec_byte = cls._wf_coef
        return n * fixed + per_col * col_bytes + per_rec * records + per_rec_byte * rec_bytes if n else 0

    @staticmethod
    def workflow_issuer(w):
        """The issuer generateWorkflowVCDocument signs with: the first record's issuer_did, the root DID without records."""
        evs = w["execution_vcs"]
        return evs[0]["issuer_did"] if evs else w["root_did"]

    @staticmethod
    def pack_workflow_requests(workflows):
        """generateWorkflowVCDocument inputs (the dicts of services.VCService.issue_workflow_vc_batch: workflow_id, execution_vcs of vc_id,
        session_id, status, created_at (an aware datetime), issuer_did; root_did, vc_id, issuance_date, snapshot_time, proof_created) -> the
        host arrays of afc_vc_issue_workflow_batch: (cols, col_off, rec_off, rec_cols, rec_col_off, created_at).  Strings are UTF-8 with lone surrogates kept as their three bytes; bytes pass as they are."""
        def b(v):
            return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)
        flat, rflat, created, counts = [], [], [], []
        for w in workflows:
            evs = w["execution_vcs"]
            flat += [b(w["workflow_id"]), b(evs[0]["session_id"] if evs else ""), b(ExpandedKeys.workflow_issuer(w)), b(w["vc_id"]),
                     b(w["issuance_date"]), b(w["snapshot_time"]), b(w["proof_created"])]
            for v in evs:
                rflat += [b(v["vc_id"]), b(v["status"])]
                created += unix_pair(v["created_at"])
            counts.append(len(evs))
        cols, col_off = pack(flat)
        rec_cols, rec_col_off = pack(rflat)
        rec_off = np.zeros(len(workflows) + 1, dtype=np.uint64)
        rec_off[1:] = np.cumsum(counts, dtype=np.uint64)
        return cols, col_off, rec_off, rec_cols, rec_col_off, np.array(created, dtype=np.int64)

    def issue_workflow_packed(self, key_index, cols, col_off, rec_off, rec_cols, rec_col_off, created_at, expanded=None):
        """afc_vc_issue_workflow_batch on host arrays (the layout of pack_workflow_requests).  Returns (docs uint8, doc_off uint64 [n+1],
        proof_values uint8 [n, 86], state uint8 [n], summary uint32 [n, 4])."""
        n = len(key_index)
        exp = self._expanded if expanded is None else expanded
        lib = _abi.load()
        cap = lib.afc_vc_workflow_bound(_abi.ptr(col_off), _abi.ptr(rec_off), _abi.ptr(rec_col_off), n)
        docs = np.empty(max(cap, 1), dtype=np.uint8)
        doc_off = np.zeros(n + 1, dtype=np.uint64)
        pv = np.empty((n, 86), dtype=np.uint8)
        state = np.empty(n, dtype=np.uint8)
        summary = np.empty((n, 4), dtype=np.uint32)
        _abi.check(lib.afc_vc_issue_workflow_batch(self.ctx.handle, _abi.ptr(exp), exp.shape[0], _abi.ptr(key_index), _abi.ptr(cols),
                                                   _abi.ptr(col_off), _abi.ptr(rec_off), _abi.ptr(rec_cols), _abi.ptr(rec_col_off),
                                                   _abi.ptr(created_at), n, _abi.ptr(docs), cap, _abi.ptr(doc_off), _abi.ptr(pv), _abi.ptr(state),
                                                   _abi.ptr(summary)), self.ctx.handle)
        return docs[:int(doc_off[n])], doc_off, pv, state, summary

    def issue_workflow_dev(self, d_key_index, d_cols, d_col_off, d_rec_off, d_rec_cols, d_rec_col_off, d_created_at, n, stream=None, d_expanded=None):
        """afc_vc_issue_workflow_batch_dev: n workflows on the device.  d_key_index: int32 [n] into this cache (or into d_expanded, K x 96);
        d_cols / d_col_off: uint8 columns and int64 [7n+1] absolute offsets (_abi.WORKFLOW_COLUMNS order); d_rec_off: int64 [n+1] absolute
        record indices; d_rec_cols / d_rec_col_off: the records' vc_id and status, int64 [2 per record + 1]; d_created_at: int64 [2 per
        record] (Unix seconds, nanoseconds).  Returns (d_docs uint8, d_doc_off int64 [n+1], d_proof_values uint8 [n, 86], d_state uint8 [n],
        d_summary int32 [n, 4], to be read as uint32)."""
        import torch
        dev = d_col_off.device
        if d_expanded is None:
            d_expanded = torch.from_numpy(self._expanded).to(dev)
        if n:
            r0, r1 = int(d_rec_off[0]), int(d_rec_off[n])
            cap = self._workflow_bound(n, int(d_col_off[n * len(_abi.WORKFLOW_COLUMNS)]) - int(d_col_off[0]), r1 - r0,
                                       int(d_rec_col_off[2 * r1]) - int(d_rec_col_off[2 * r0]))
        else:
            cap = 0
        d_docs = torch.empty(max(cap, 1), dtype=torch.uint8, device=dev)
        d_doc_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_pv = torch.empty((n, 86), dtype=torch.uint8, device=dev)
        d_state = torch.empty(n, dtype=torch.uint8, device=dev)
        d_summary = torch.empty((n, 4), dtype=torch.int32, device=dev)
        _abi.check(_abi.load().afc_vc_issue_workflow_batch_dev(self.ctx.handle, _abi.ptr(d_expanded), d_expanded.shape[0], _abi.ptr(d_key_index),
                                                               _abi.ptr(d_cols), _abi.ptr(d_col_off), _abi.ptr(d_rec_off), _abi.ptr(d_rec_cols),
                                                               _abi.ptr(d_rec_col_off), _abi.ptr(d_created_at), n, _abi.ptr(d_docs), cap,
                                                               _abi.ptr(d_doc_off), _abi.ptr(d_pv), _abi.ptr(d_state), _abi.ptr(d_summary),
                                                               self.ctx._stream(stream)), self.ctx.handle)
        total = int(d_doc_off[n]) if n else 0
        return d_docs[:total], d_doc_off, d_pv, d_state, d_summary

    def issue_workflows(self, workflows):
        """generateWorkflowVCDocument for many workflows in one host-buffer call: [{"vc_document": bytes, "signature": str, "state": int,
        "summary": [status id, completed, start record, end record]}] (an AFC_WORKFLOW_HOST workflow has an empty document and signature)."""
        n = len(workflows)
        if n == 0:
            return []
        ki = self.key_index([self.workflow_issuer(w) for w in workflows])
        docs, off, pv, state, summ = self.issue_workflow_packed(ki, *self.pack_workflow_requests(workflows))
        buf = docs.tobytes()
        return [{"vc_document": buf[int(off[i]):int(off[i + 1])], "signature": pv[i].tobytes().decode() if state[i] == _abi.WORKFLOW_BUILT else "",
                 "state": int(state[i]), "summary": [int(x) for x in summ[i]]} for i in range(n)]

    # -- workflow VC chains (afc_vc_workflow_chain_batch)
    @staticmethod
    def pack_chain_requests(workflows):
        """GetWorkflowVCChain inputs: the dicts of services.VCService.get_workflow_vc_chain_batch (those of issue_workflow_vc_batch, each
        ExecutionVC record complete: execution_id, workflow_id, session_id, agent_node_id / workflow_name (None = nil), issuer_did,
        target_did, caller_did, vc_document (bytes, None = nil), signature, storage_uri, document_size_bytes, input_hash, output_hash,
        status, created_at (an aware datetime); plus workflow_vc_id, resolved_at and snapshot, an aware datetime) -> the host arrays of
        afc_vc_workflow_chain_batch after key_index: pack_workflow_requests's six, then chain_cols, chain_col_off, clock, chain_rec_cols,
        chain_rec_col_off, rec_flags, doc_size, created_off."""
        def b(v):
            return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)
        wcols, rcols, clock, flags, size, zone = [], [], [], [], [], []
        for w in workflows:
            wcols += [b(w["workflow_vc_id"]), b(w["resolved_at"])]
            clock += unix_pair(w["snapshot"]) + [zone_seconds(w["snapshot"])]
            for v in w["execution_vcs"]:
                f = 0
                for key, bit in (("agent_node_id", _abi.CHAIN_AGENT_NODE_ID_NIL), ("workflow_name", _abi.CHAIN_WORKFLOW_NAME_NIL),
                                 ("vc_document", _abi.CHAIN_VC_DOCUMENT_NIL)):
                    if v.get(key) is None:
                        f |= bit
                rcols += [b(v.get(k) or b"") for k in _abi.CHAIN_RECORD_COLUMNS]
                flags.append(f)
                size.append(int(v["document_size_bytes"]))
                zone.append(zone_seconds(v["created_at"]))
        chain_cols, chain_col_off = pack(wcols)
        chain_rec_cols, chain_rec_col_off = pack(rcols)
        return (*ExpandedKeys.pack_workflow_requests(workflows), chain_cols, chain_col_off, np.array(clock, dtype=np.int64), chain_rec_cols,
                chain_rec_col_off, np.array(flags + [0], dtype=np.uint8), np.array(size + [0], dtype=np.int64), np.array(zone + [0], dtype=np.int32))

    _chain_coef = None

    @classmethod
    def _chain_bound(cls, n, col_bytes, records, rec_bytes, chain_col_bytes, chain_rec_bytes):
        """afc_vc_workflow_chain_bound for n workflows with these totals.  The library needs offset arrays that span the batch's records,
        which the device call only has on the device; the bound is linear in the six totals, so its coefficients are read off the library
        once, with one-workflow arrays (tests/test_vcchain_hostsim.py holds this equal to the library's bound)."""
        if cls._chain_coef is None:
            lib = _abi.load()
            a = [np.zeros(len(_abi.WORKFLOW_COLUMNS) + 1, dtype=np.uint64), np.zeros(2, dtype=np.uint64), np.zeros(3, dtype=np.uint64),
                 np.zeros(3, dtype=np.uint64), np.zeros(len(_abi.CHAIN_RECORD_COLUMNS) + 1, dtype=np.uint64)]

            def f(k=None, at=None):
                if k is not None:
                    a[k][at] = 1
                v = lib.afc_vc_workflow_chain_bound(*[_abi.ptr(x) for x in a], 1)
                if k is not None and k != 1:
                    a[k][at] = 0
                return v
            fixed = f()
            per_col, per_ccol = f(0, -1) - fixed, f(3, -1) - fixed
            per_rec = f(1, 1) - fixed                                  # rec_off stays [0, 1] for the two per-record-byte probes
            cls._chain_coef = (fixed, per_col, per_rec, f(2, 2) - fixed - per_rec, per_ccol, f(4, -1) - fixed - per_rec)
        c = cls._chain_coef
        return n * c[0] + c[1] * col_bytes + c[2] * records + c[3] * rec_bytes + c[4] * chain_col_bytes + c[5] * chain_rec_bytes if n else 0

    @classmethod
    def _chain_bound_dev(cls, n, d_col_off, d_rec_off, d_rec_col_off, d_ccol_off, d_crcol_off):
        """_chain_bound of device offset arrays: their ten ends in one device-to-host copy."""
        import torch
        C, RC = len(_abi.WORKFLOW_COLUMNS), len(_abi.CHAIN_RECORD_COLUMNS)
        at = lambda t, k: t[k:k + 1]                                # views: no index tensor crosses to the device
        r = torch.cat([at(d_rec_off, 0), at(d_rec_off, n)])
        e = [int(x) for x in torch.cat([at(d_col_off, 0), at(d_col_off, C * n), r, d_rec_col_off.index_select(0, 2 * r), at(d_ccol_off, 0),
                                        at(d_ccol_off, 2 * n), d_crcol_off.index_select(0, RC * r)]).cpu().tolist()]
        span = lambda lo, hi: max(hi - lo, 0)
        return cls._chain_bound(n, span(e[0], e[1]), span(e[2], e[3]), span(e[4], e[5]), span(e[6], e[7]), span(e[8], e[9]))

    def workflow_chain_packed(self, directory, key_index, *arrays, expanded=None):
        """afc_vc_workflow_chain_batch on host arrays (the layout of pack_chain_requests).  Returns (bodies uint8, body_off uint64 [n+1],
        state uint8 [n])."""
        n = len(key_index)
        cols, col_off, rec_off, rec_cols, rec_col_off, created, chain_cols, chain_col_off, clock, crec_cols, crec_col_off, flags, size, zone = arrays
        created = np.ascontiguousarray(created if len(created) else np.zeros(2, dtype=np.int64))
        exp = self._expanded if expanded is None else expanded
        lib = _abi.load()
        cap = lib.afc_vc_workflow_chain_bound(_abi.ptr(col_off), _abi.ptr(rec_off), _abi.ptr(rec_col_off), _abi.ptr(chain_col_off),
                                              _abi.ptr(crec_col_off), n)
        bodies = np.empty(max(cap, 1), dtype=np.uint8)
        body_off = np.zeros(n + 1, dtype=np.uint64)
        state = np.empty(max(n, 1), dtype=np.uint8)
        _abi.check(lib.afc_vc_workflow_chain_batch(self.ctx.handle, _abi.ptr(exp), exp.shape[0], _abi.ptr(key_index), _abi.ptr(cols),
                                                   _abi.ptr(col_off), _abi.ptr(rec_off), _abi.ptr(rec_cols), _abi.ptr(rec_col_off), _abi.ptr(created),
                                                   _abi.ptr(chain_cols), _abi.ptr(chain_col_off), _abi.ptr(clock), _abi.ptr(crec_cols),
                                                   _abi.ptr(crec_col_off), _abi.ptr(flags), _abi.ptr(size), _abi.ptr(zone), directory.handle, n,
                                                   _abi.ptr(bodies), cap, _abi.ptr(body_off), _abi.ptr(state)), self.ctx.handle)
        return bodies[:int(body_off[n])], body_off, state[:n]

    def workflow_chain_dev(self, directory, d_key_index, d_arrays, n, stream=None, d_expanded=None):
        """afc_vc_workflow_chain_batch_dev: d_arrays are the 14 arrays of pack_chain_requests on the device (offsets as int64, uint32
        arrays as int32).  Returns (d_bodies uint8, d_body_off int64 [n+1], d_state uint8 [n])."""
        import torch
        d_cols, d_col_off, d_rec_off, d_rec_cols, d_rec_col_off, d_created, d_ccols, d_ccol_off, d_clock, d_crcols, d_crcol_off, d_flags, d_size, d_zone = d_arrays
        dev = d_col_off.device
        if d_expanded is None:
            d_expanded = torch.from_numpy(self._expanded).to(dev)
        lib = _abi.load()
        cap = self._chain_bound_dev(n, d_col_off, d_rec_off, d_rec_col_off, d_ccol_off, d_crcol_off) if n else 0
        d_bodies = torch.empty(max(cap, 1), dtype=torch.uint8, device=dev)
        d_body_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_state = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        _abi.check(lib.afc_vc_workflow_chain_batch_dev(self.ctx.handle, _abi.ptr(d_expanded), d_expanded.shape[0], _abi.ptr(d_key_index),
                                                       *[_abi.ptr(t) for t in d_arrays], directory.handle, n, _abi.ptr(d_bodies), cap,
                                                       _abi.ptr(d_body_off), _abi.ptr(d_state), self.ctx._stream(stream)), self.ctx.handle)
        total = int(d_body_off[n]) if n else 0
        return d_bodies[:total], d_body_off, d_state[:n]

    def workflow_chains(self, workflows, directory):
        """GetWorkflowVCChain + c.JSON for many workflows in one host-buffer call: [(state, body bytes)] (an AFC_CHAIN_HOST workflow has an
        empty body)."""
        if not workflows:
            return []
        ki = self.key_index([self.workflow_issuer(w) for w in workflows])
        bodies, off, state = self.workflow_chain_packed(directory, ki, *self.pack_chain_requests(workflows))
        buf = bodies.tobytes()
        return [(int(state[i]), buf[int(off[i]):int(off[i + 1])]) for i in range(len(workflows))]

    # -- agent DID registration (afc_did_register_batch)
    def _append(self, expanded, dids):
        base = self._expanded.shape[0]
        self._expanded = np.concatenate([self._expanded, expanded])
        for i, d in enumerate(dids):
            self._index[d] = base + i

    @staticmethod
    def pack_register_requests(requests):
        """DIDRegistrationRequests ({"agent_node_id", "reasoners": [ids], "skills": [ids]}; str or bytes, str as UTF-8 with lone surrogates
        kept as their three bytes) -> the host arrays of afc_did_register_batch: (node_ids, node_off, id_idx, ids, id_off)."""
        def b(v):
            return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)
        flat, idx = [], [0]
        for r in requests:
            flat += [b(x) for x in r.get("reasoners") or ()]
            idx.append(len(flat))
            flat += [b(x) for x in r.get("skills") or ()]
            idx.append(len(flat))
        nodes, node_off = pack([b(r["agent_node_id"]) for r in requests])
        ids, id_off = pack(flat)
        return nodes, node_off, np.array(idx, dtype=np.uint64), ids, id_off

    def register_packed(self, master_seed, server_id, node_ids, node_off, agent_index, id_idx, ids, id_off, append=True):
        """afc_did_register_batch on host arrays (the layout of pack_register_requests; agent_index uint32 [n]).  Returns a dict: comp_off
        uint64 [n+1], expanded uint8 [C, 96], pks [C, 32], dids [C, 55], paths [C, 48], flags uint8 [C] (_abi.DID_KEPT), body uint8,
        body_off uint64 [n+1], for the C = comp_off[n] components.  With append the expanded keys join this cache under their DIDs."""
        n = len(agent_index)
        sid = server_id.encode() if isinstance(server_id, str) else bytes(server_id)
        if len(master_seed) != 32:
            raise ValueError("the master seed is 32 bytes")
        lib = _abi.load()
        m = int(id_idx[2 * n]) - int(id_idx[0]) if n else 0
        S = n + m
        cap = lib.afc_did_register_bound(_abi.ptr(node_off), _abi.ptr(id_idx), _abi.ptr(id_off), n, len(sid))
        out = {"comp_off": np.zeros(n + 1, dtype=np.uint64), "expanded": np.empty((S, 96), dtype=np.uint8), "pks": np.empty((S, 32), dtype=np.uint8),
               "dids": np.empty((S, _abi.DID_CHARS), dtype=np.uint8), "paths": np.empty((S, _abi.DID_PATH_SLOT), dtype=np.uint8),
               "flags": np.empty(S, dtype=np.uint8), "body": np.empty(max(cap, 1), dtype=np.uint8), "body_off": np.zeros(n + 1, dtype=np.uint64)}
        ms = np.frombuffer(bytes(master_seed), dtype=np.uint8).copy()
        ai = np.ascontiguousarray(agent_index, dtype=np.uint32)
        _abi.check(lib.afc_did_register_batch(self.ctx.handle, _abi.ptr(ms), sid, len(sid), _abi.ptr(node_ids), _abi.ptr(node_off), _abi.ptr(ai),
                                              _abi.ptr(id_idx), _abi.ptr(ids), _abi.ptr(id_off), n, _abi.ptr(out["comp_off"]), _abi.ptr(out["expanded"]),
                                              _abi.ptr(out["pks"]), _abi.ptr(out["dids"]), _abi.ptr(out["paths"]), _abi.ptr(out["flags"]),
                                              _abi.ptr(out["body"]), cap, _abi.ptr(out["body_off"])), self.ctx.handle)
        ms[:] = 0
        C_ = int(out["comp_off"][n])
        for k in ("expanded", "pks", "dids", "paths", "flags"):
            out[k] = out[k][:C_]
        out["body"] = out["body"][:int(out["body_off"][n])]
        if append:
            self._append(out["expanded"], [d.tobytes().decode() for d in out["dids"]])
        return out

    def register_dev(self, d_master_seed, server_id, d_node_ids, d_node_off, d_agent_index, d_id_idx, d_ids, d_id_off, n, stream=None, append=True):
        """afc_did_register_batch_dev: n requests on the device (int64 offset arrays, int32 agent indices, a 32-byte uint8 master seed).
        Returns a dict of device tensors as register_packed returns arrays, each cut to the C components (comp_off, body_off int64).  With
        append the expanded keys are copied into this cache under their DIDs."""
        import torch
        dev = d_node_off.device
        sid = server_id.encode() if isinstance(server_id, str) else bytes(server_id)
        lib = _abi.load()
        if n:
            r0, r1 = int(d_id_idx[0]), int(d_id_idx[2 * n])
            m = r1 - r0
            node_bytes = int(d_node_off[n]) - int(d_node_off[0])
            ends = np.array([0, node_bytes], dtype=np.uint64)
            idx = np.array([0, 0, m], dtype=np.uint64)
            off = np.zeros(m + 1, dtype=np.uint64)
            off[m] = int(d_id_off[r1]) - int(d_id_off[r0])
            cap = lib.afc_did_register_bound(_abi.ptr(ends), _abi.ptr(idx), _abi.ptr(off), 1, len(sid))
            cap += (n - 1) * lib.afc_did_register_bound(_abi.ptr(np.zeros(2, dtype=np.uint64)), _abi.ptr(np.zeros(3, dtype=np.uint64)),
                                                        _abi.ptr(np.zeros(1, dtype=np.uint64)), 1, len(sid))
        else:
            m, cap = 0, 0
        S = n + m
        out = {"comp_off": torch.zeros(n + 1, dtype=torch.int64, device=dev), "expanded": torch.empty((S, 96), dtype=torch.uint8, device=dev),
               "pks": torch.empty((S, 32), dtype=torch.uint8, device=dev), "dids": torch.empty((S, _abi.DID_CHARS), dtype=torch.uint8, device=dev),
               "paths": torch.empty((S, _abi.DID_PATH_SLOT), dtype=torch.uint8, device=dev), "flags": torch.empty(S, dtype=torch.uint8, device=dev),
               "body": torch.empty(max(cap, 1), dtype=torch.uint8, device=dev), "body_off": torch.zeros(n + 1, dtype=torch.int64, device=dev)}
        _abi.check(lib.afc_did_register_batch_dev(self.ctx.handle, _abi.ptr(d_master_seed), sid, len(sid), _abi.ptr(d_node_ids), _abi.ptr(d_node_off),
                                                  _abi.ptr(d_agent_index), _abi.ptr(d_id_idx), _abi.ptr(d_ids), _abi.ptr(d_id_off), n,
                                                  _abi.ptr(out["comp_off"]), _abi.ptr(out["expanded"]), _abi.ptr(out["pks"]), _abi.ptr(out["dids"]),
                                                  _abi.ptr(out["paths"]), _abi.ptr(out["flags"]), _abi.ptr(out["body"]), cap, _abi.ptr(out["body_off"]),
                                                  self.ctx._stream(stream)), self.ctx.handle)
        if n:
            C_ = int(out["comp_off"][n])
            for k in ("expanded", "pks", "dids", "paths", "flags"):
                out[k] = out[k][:C_]
            out["body"] = out["body"][:int(out["body_off"][n])]
        if append and n:
            self._append(out["expanded"].cpu().numpy(), [d.tobytes().decode() for d in out["dids"].cpu().numpy()])
        return out

    def register(self, master_seed, server_id, requests, agent_base):
        """handleNewRegistration for many new agents in one host-buffer call; request k gets agent index agent_base + k.  Returns per
        request {"body": the DIDRegistrationResponse bytes, "components": [{"did", "pk", "path", "type", "id", "kept"}]} (agent first,
        then the non-empty reasoner ids, then the non-empty skill ids, in request order)."""
        n = len(requests)
        if n == 0:
            return []
        nodes, node_off, id_idx, ids, id_off = self.pack_register_requests(requests)
        ai = np.arange(agent_base, agent_base + n, dtype=np.uint64).astype(np.uint32)
        R = self.register_packed(master_seed, server_id, nodes, node_off, ai, id_idx, ids, id_off)
        body = R["body"].tobytes()
        out = []
        for i, r in enumerate(requests):
            c0, c1 = int(R["comp_off"][i]), int(R["comp_off"][i + 1])
            kinds = [("agent", r["agent_node_id"])] + [("reasoner", x) for x in r.get("reasoners") or () if len(x)] + \
                    [("skill", x) for x in r.get("skills") or () if len(x)]
            comps = [{"did": R["dids"][c].tobytes().decode(), "pk": R["pks"][c].tobytes(), "path": R["paths"][c].tobytes().rstrip(b"\0").decode(),
                      "type": t, "id": x, "kept": bool(R["flags"][c] & _abi.DID_KEPT)} for c, (t, x) in zip(range(c0, c1), kinds)]
            out.append({"body": body[int(R["body_off"][i]):int(R["body_off"][i + 1])], "components": comps})
        return out

    # -- known agents re-registered (afc_did_reregister_batch)
    REREG_COLUMNS = ("did", "public_key_jwk", "derivation_path", "function_name")

    @staticmethod
    def pack_reregister_requests(requests):
        """Re-registrations of known agents ({"agent": {"did", "public_key_jwk", "derivation_path", "reasoners", "skills"}, "reasoners":
        [ids], "skills": [ids]}; the agent's "reasoners" and "skills" map each key to {"did", "public_key_jwk", "derivation_path",
        "function_name"}, as a dict or as (key, value) pairs; str or bytes as in pack_register_requests) -> the host arrays of
        afc_did_reregister_batch: (agent_cols, agent_col_off, id_idx, ids, id_off, reg_idx, reg_cols, reg_col_off)."""
        def b(v):
            return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)

        def pairs(m):
            return list(m.items()) if isinstance(m, dict) else list(m)
        acols, flat, idx, rflat, ridx = [], [], [0], [], [0]
        for r in requests:
            a = r["agent"]
            acols += [b(a["did"]), b(a["public_key_jwk"]), b(a["derivation_path"])]
            for kind in ("reasoners", "skills"):
                flat += [b(x) for x in r.get(kind) or ()]
                idx.append(len(flat))
                for key, c in pairs(a.get(kind) or ()):
                    rflat += [b(key)] + [b(c.get(k) or b"") for k in ExpandedKeys.REREG_COLUMNS]
                ridx.append(len(rflat) // 5)
        agent_cols, agent_col_off = pack(acols)
        ids, id_off = pack(flat)
        reg_cols, reg_col_off = pack(rflat)
        return (agent_cols, agent_col_off, np.array(idx, dtype=np.uint64), ids, id_off, np.array(ridx, dtype=np.uint64), reg_cols, reg_col_off)

    def _append_slots(self, state, counts, expanded, dids):
        """The key slots that received a new component join this cache under their DIDs."""
        n = len(state)
        live = [t for t in range(2 * n) if state[t >> 1] == _abi.DIDRR_PARTIAL and counts[t >> 1][t & 1]]
        if live:
            self._append(expanded[live], [dids[t].tobytes().decode() for t in live])

    def reregister_packed(self, master_seed, server_id, agent_cols, agent_col_off, agent_index, id_idx, ids, id_off, reg_idx, reg_cols, reg_col_off,
                          append=True):
        """afc_did_reregister_batch on host arrays (the layout of pack_reregister_requests; agent_index uint32 [n]).  Returns a dict: state
        uint8 [n] (_abi.DIDRR_*), counts uint32 [n, 4], expanded uint8 [2n, 96], pks [2n, 32], dids [2n, 55], paths [2n, 48] (key slot 2i + 0
        for reasoners, 2i + 1 for skills), reg_flags uint8 [G] (_abi.DIDRR_GONE), id_flags uint8 [m] (_abi.DIDRR_NEW | _abi.DID_KEPT), body
        uint8, body_off uint64 [n+1].  With append the keys of the slots in use join this cache under their DIDs."""
        n = len(agent_index)
        sid = server_id.encode() if isinstance(server_id, str) else bytes(server_id)
        if len(master_seed) != 32:
            raise ValueError("the master seed is 32 bytes")
        lib = _abi.load()
        m = int(id_idx[2 * n]) - int(id_idx[0]) if n else 0
        G = int(reg_idx[2 * n]) - int(reg_idx[0]) if n else 0
        cap = lib.afc_did_reregister_bound(_abi.ptr(agent_col_off), _abi.ptr(id_idx), _abi.ptr(id_off), _abi.ptr(reg_idx), _abi.ptr(reg_col_off), n,
                                           len(sid))
        out = {"state": np.zeros(n, dtype=np.uint8), "counts": np.zeros((n, 4), dtype=np.uint32), "expanded": np.empty((2 * n, 96), dtype=np.uint8),
               "pks": np.empty((2 * n, 32), dtype=np.uint8), "dids": np.empty((2 * n, _abi.DID_CHARS), dtype=np.uint8),
               "paths": np.empty((2 * n, _abi.DID_PATH_SLOT), dtype=np.uint8), "reg_flags": np.zeros(G, dtype=np.uint8),
               "id_flags": np.zeros(m, dtype=np.uint8), "body": np.empty(max(cap, 1), dtype=np.uint8), "body_off": np.zeros(n + 1, dtype=np.uint64)}
        ms = np.frombuffer(bytes(master_seed), dtype=np.uint8).copy()
        ai = np.ascontiguousarray(agent_index, dtype=np.uint32)
        _abi.check(lib.afc_did_reregister_batch(self.ctx.handle, _abi.ptr(ms), sid, len(sid), _abi.ptr(agent_cols), _abi.ptr(agent_col_off), _abi.ptr(ai),
                                                _abi.ptr(id_idx), _abi.ptr(ids), _abi.ptr(id_off), _abi.ptr(reg_idx), _abi.ptr(reg_cols),
                                                _abi.ptr(reg_col_off), n, _abi.ptr(out["state"]), _abi.ptr(out["counts"]), _abi.ptr(out["expanded"]),
                                                _abi.ptr(out["pks"]), _abi.ptr(out["dids"]), _abi.ptr(out["paths"]), _abi.ptr(out["reg_flags"]),
                                                _abi.ptr(out["id_flags"]), _abi.ptr(out["body"]), cap, _abi.ptr(out["body_off"])), self.ctx.handle)
        ms[:] = 0
        out["body"] = out["body"][:int(out["body_off"][n])]
        if append:
            self._append_slots(out["state"], out["counts"], out["expanded"], out["dids"])
        return out

    def reregister_dev(self, d_master_seed, server_id, d_agent_cols, d_agent_col_off, d_agent_index, d_id_idx, d_ids, d_id_off, d_reg_idx, d_reg_cols,
                       d_reg_col_off, n, stream=None, append=True):
        """afc_did_reregister_batch_dev: n requests on the device (int64 offset arrays, int32 agent indices, a 32-byte uint8 master seed).
        Returns a dict of device tensors as reregister_packed returns arrays (body_off int64, counts int32).  With append the keys of the
        slots in use are copied into this cache under their DIDs."""
        import torch
        dev = d_agent_col_off.device
        sid = server_id.encode() if isinstance(server_id, str) else bytes(server_id)
        lib = _abi.load()
        m = G = cap = 0
        if n:
            r0, r1, g0, g1 = int(d_id_idx[0]), int(d_id_idx[2 * n]), int(d_reg_idx[0]), int(d_reg_idx[2 * n])
            m, G = r1 - r0, g1 - g0
            aoff = np.array([0, 0, 0, int(d_agent_col_off[3 * n]) - int(d_agent_col_off[0])], dtype=np.uint64)
            ioff = np.zeros(m + 1, dtype=np.uint64)
            ioff[m] = int(d_id_off[r1]) - int(d_id_off[r0])
            roff = np.zeros(5 * G + 1, dtype=np.uint64)
            roff[5 * G] = int(d_reg_col_off[5 * g1]) - int(d_reg_col_off[5 * g0])
            iidx, ridx = np.array([0, 0, m], dtype=np.uint64), np.array([0, 0, G], dtype=np.uint64)
            zero = np.zeros(4, dtype=np.uint64)                   # an empty request: every end 0
            cap = lib.afc_did_reregister_bound(_abi.ptr(aoff), _abi.ptr(iidx), _abi.ptr(ioff), _abi.ptr(ridx), _abi.ptr(roff), 1, len(sid))
            cap += (n - 1) * lib.afc_did_reregister_bound(*[_abi.ptr(zero)] * 5, 1, len(sid))
        e = lambda shape, dt=torch.uint8: torch.empty(shape, dtype=dt, device=dev)  # noqa: E731
        out = {"state": e(n), "counts": e((n, 4), torch.int32), "expanded": e((2 * n, 96)), "pks": e((2 * n, 32)), "dids": e((2 * n, _abi.DID_CHARS)),
               "paths": e((2 * n, _abi.DID_PATH_SLOT)), "reg_flags": e(G), "id_flags": e(m), "body": e(max(cap, 1)),
               "body_off": torch.zeros(n + 1, dtype=torch.int64, device=dev)}
        _abi.check(lib.afc_did_reregister_batch_dev(self.ctx.handle, _abi.ptr(d_master_seed), sid, len(sid), _abi.ptr(d_agent_cols),
                                                    _abi.ptr(d_agent_col_off), _abi.ptr(d_agent_index), _abi.ptr(d_id_idx), _abi.ptr(d_ids),
                                                    _abi.ptr(d_id_off), _abi.ptr(d_reg_idx), _abi.ptr(d_reg_cols), _abi.ptr(d_reg_col_off), n,
                                                    _abi.ptr(out["state"]), _abi.ptr(out["counts"]), _abi.ptr(out["expanded"]), _abi.ptr(out["pks"]),
                                                    _abi.ptr(out["dids"]), _abi.ptr(out["paths"]), _abi.ptr(out["reg_flags"]), _abi.ptr(out["id_flags"]),
                                                    _abi.ptr(out["body"]), cap, _abi.ptr(out["body_off"]), self.ctx._stream(stream)), self.ctx.handle)
        if n:
            out["body"] = out["body"][:int(out["body_off"][n])]
            if append:
                self._append_slots(out["state"].cpu().numpy(), out["counts"].cpu().numpy(), out["expanded"].cpu().numpy(), out["dids"].cpu().numpy())
        return out

    @staticmethod
    def agent_index_of(derivation_path):
        """The <a> of an agent's stored path m/44'/<h>'/<a>': the index its new components' paths take (the reference's own choice, the
        agent's place in Go's randomised map iteration, changes from run to run)."""
        p = derivation_path.decode() if isinstance(derivation_path, (bytes, bytearray)) else derivation_path
        parts = p.split("/")
        if len(parts) != 4 or parts[0] != "m" or parts[1] != "44'" or not parts[3].endswith("'") or not parts[3][:-1].isdigit():
            raise ValueError("not an agent derivation path: %r" % p)
        return int(parts[3][:-1]) & 0xFFFFFFFF

    def reregister(self, master_seed, server_id, requests):
        """RegisterAgent for many known agents in one host-buffer call (pack_reregister_requests' requests; "agent_index" overrides the <a>
        read from the agent's stored path).  Returns per request {"state", "counts", "body", "gone": [reasoners, skills] of bools in the
        agent's order, "new": [reasoners, skills] of the ids the registry adds (the kept occurrences), "slots": [reasoners, skills] of None or
        {"did", "pk", "path", "public_key_jwk"}}."""
        n = len(requests)
        if n == 0:
            return []
        ai = np.array([r["agent_index"] if "agent_index" in r else self.agent_index_of(r["agent"]["derivation_path"]) for r in requests],
                      dtype=np.uint64).astype(np.uint32)
        A = self.pack_reregister_requests(requests)
        R = self.reregister_packed(master_seed, server_id, A[0], A[1], ai, *A[2:])
        body = R["body"].tobytes()
        out = []
        g = k = 0
        for i, r in enumerate(requests):
            res = {"state": int(R["state"][i]), "counts": [int(x) for x in R["counts"][i]], "body": body[int(R["body_off"][i]):int(R["body_off"][i + 1])],
                   "gone": [], "new": [], "slots": []}
            for kind in ("reasoners", "skills"):
                regs = r["agent"].get(kind) or ()
                res["gone"].append([bool(f & _abi.DIDRR_GONE) for f in R["reg_flags"][g:g + len(regs)]])
                g += len(regs)
                ids = list(r.get(kind) or ())
                fl = R["id_flags"][k:k + len(ids)]
                res["new"].append([x for x, f in zip(ids, fl) if f == _abi.DIDRR_NEW | _abi.DID_KEPT])
                k += len(ids)
            for t in (2 * i, 2 * i + 1):
                if res["state"] == _abi.DIDRR_PARTIAL and res["counts"][t & 1]:
                    pk = R["pks"][t].tobytes()
                    res["slots"].append({"did": R["dids"][t].tobytes().decode(), "pk": pk, "path": R["paths"][t].tobytes().rstrip(b"\0").decode(),
                                         "public_key_jwk": public_jwk(pk)})
                else:
                    res["slots"].append(None)
            out.append(res)
        return out


def public_jwk(pk: bytes) -> bytes:
    """The public JWK text handleNewRegistration and PartialRegisterAgent store (json.Marshal of a map: keys sorted)."""
    x = base64.urlsafe_b64encode(pk).rstrip(b"=")
    return b'{"alg":"EdDSA","crv":"Ed25519","kty":"OKP","use":"sig","x":"' + x + b'"}'


_EPOCH = datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc)


def unix_pair(t):
    """(Unix seconds, nanoseconds) of an aware datetime."""
    if t.tzinfo is None:
        raise ValueError("created_at must be an aware datetime")
    d = t - _EPOCH
    return [d.days * 86400 + d.seconds, d.microseconds * 1000]


def zone_seconds(t):
    """The UTC offset of an aware datetime in seconds."""
    return int(t.utcoffset().total_seconds())


class DIDDirectory:
    """afc_did_directory: the public half of a DID registry on the device — DIDs, their public keys and their order — for the DID
    resolution bundle of workflow chains.  No verify tables are built (a KeySet's are 384 KB per key)."""

    def __init__(self, dids, pks, ctx=None):
        self.ctx = ctx or default_context()
        self._lib = _abi.load()
        if len(dids) != len(pks) or any(len(p) != 32 for p in pks):
            raise ValueError("one 32-byte public key per DID")
        self.dids = [d.encode("utf-8", "surrogatepass") if isinstance(d, str) else bytes(d) for d in dids]
        self.pks = [bytes(p) for p in pks]
        buf, off = pack(self.dids)
        arr = np.frombuffer(b"".join(self.pks) or bytes(32), dtype=np.uint8).copy()
        h = C.c_void_p()
        _abi.check(self._lib.afc_did_directory_new(self.ctx.handle, _abi.ptr(arr), _abi.ptr(buf), _abi.ptr(off), len(self.dids), C.byref(h)),
                   self.ctx.handle)
        self.handle = h

    @staticmethod
    def _b(v):
        return v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v)

    def set_identities(self, kinds, paths, function_names, jwks):
        """afc_did_directory_set_identities: per DID, in the directory's order, its kind (_abi.DID_KIND_*), derivation path, function name
        and stored public JWK text (str or bytes).  Once per directory."""
        n = len(self.dids)
        if not len(kinds) == len(paths) == len(function_names) == len(jwks) == n:
            raise ValueError("one kind, path, function name and JWK per DID")
        cols = []
        for p, f, j in zip(paths, function_names, jwks):
            cols += [self._b(p), self._b(f), self._b(j)]
        buf, off = pack(cols)
        k = np.array(list(kinds) + [0], dtype=np.uint8)
        _abi.check(self._lib.afc_did_directory_set_identities(self.handle, _abi.ptr(k), _abi.ptr(buf), _abi.ptr(off)), self.ctx.handle)

    @classmethod
    def pack_requests(cls, requests):
        """[(kind, did)] (kind _abi.DIDRES_RESOLVE or _DOCUMENT; did str or bytes) -> (kinds uint8, reqs, req_off)."""
        reqs, req_off = pack([cls._b(d) for _, d in requests])
        return np.array([k for k, _ in requests] + [0], dtype=np.uint8), reqs, req_off

    def _bound(self, n, req_bytes):
        """afc_did_resolve_bound for n requests of req_bytes bytes: it is linear in both, read off the library with one-request arrays."""
        per = self._lib.afc_did_resolve_bound(self.handle, _abi.ptr(np.zeros(2, dtype=np.uint64)), 1)
        per_byte = self._lib.afc_did_resolve_bound(self.handle, _abi.ptr(np.array([0, 1], dtype=np.uint64)), 1) - per
        return n * per + per_byte * req_bytes if n else 0

    def resolve_packed(self, kinds, reqs, req_off):
        """afc_did_resolve_batch on host arrays (pack_requests).  Returns (bodies uint8, body_off uint64 [n+1], state uint8 [n])."""
        n = len(req_off) - 1
        cap = self._lib.afc_did_resolve_bound(self.handle, _abi.ptr(req_off), n)
        bodies = np.empty(max(cap, 1), dtype=np.uint8)
        body_off = np.zeros(n + 1, dtype=np.uint64)
        state = np.empty(max(n, 1), dtype=np.uint8)
        _abi.check(self._lib.afc_did_resolve_batch(self.ctx.handle, self.handle, _abi.ptr(kinds), _abi.ptr(reqs), _abi.ptr(req_off), n,
                                                   _abi.ptr(bodies), cap, _abi.ptr(body_off), _abi.ptr(state)), self.ctx.handle)
        return bodies[:int(body_off[n])], body_off, state[:n]

    def resolve_dev(self, d_kinds, d_reqs, d_req_off, n, stream=None):
        """afc_did_resolve_batch_dev on device tensors (kinds uint8, request bytes uint8, offsets int64 [n+1]).  Returns (d_bodies uint8,
        d_body_off int64 [n+1], d_state uint8 [n])."""
        import torch
        dev = d_req_off.device
        cap = 0
        if n:
            a, b = (int(x) for x in torch.cat([d_req_off[0:1], d_req_off[n:n + 1]]).cpu().tolist())
            cap = self._bound(n, max(b - a, 0))
        d_bodies = torch.empty(max(cap, 1), dtype=torch.uint8, device=dev)
        d_body_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_state = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        _abi.check(self._lib.afc_did_resolve_batch_dev(self.ctx.handle, self.handle, _abi.ptr(d_kinds), _abi.ptr(d_reqs), _abi.ptr(d_req_off), n,
                                                       _abi.ptr(d_bodies), cap, _abi.ptr(d_body_off), _abi.ptr(d_state), self.ctx._stream(stream)),
                   self.ctx.handle)
        total = int(d_body_off[n]) if n else 0
        return d_bodies[:total], d_body_off, d_state[:n]

    def resolve(self, requests):
        """Both DID handlers for many requests in one host-buffer call: [(state, body bytes)] in request order (an AFC_DIDRES_HOST request
        has an empty body)."""
        if not requests:
            return []
        bodies, off, state = self.resolve_packed(*self.pack_requests(requests))
        buf = bodies.tobytes()
        return [(int(state[i]), buf[int(off[i]):int(off[i + 1])]) for i in range(len(requests))]

    def close(self):
        if getattr(self, "handle", None):
            self._lib.afc_did_directory_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class KeySet:
    """afc_keyset: issuer public keys with device-resident verification tables (384 KB per key).  With `dids` (one per key) the
    set also resolves issuers by DID on the device, which the stored-document verification (verify_stored) needs."""

    def __init__(self, pks, ctx=None, dids=None):
        self.ctx = ctx or default_context()
        self._lib = _abi.load()
        for p in pks:
            if len(p) != 32:
                raise ValueError("ed25519: bad public key length: %d" % len(p))        # Go panics
        self.pks = [bytes(p) for p in pks]
        arr = np.frombuffer(b"".join(self.pks), dtype=np.uint8).reshape(-1, 32).copy()
        h = C.c_void_p()
        if dids is None:
            self.dids = None
            _abi.check(self._lib.afc_keyset_new(self.ctx.handle, _abi.ptr(arr), arr.shape[0], C.byref(h)), self.ctx.handle)
        else:
            if len(dids) != len(self.pks):
                raise ValueError("one DID per key")
            self.dids = [d.encode() if isinstance(d, str) else bytes(d) for d in dids]
            buf, off = pack(self.dids)
            _abi.check(self._lib.afc_keyset_new_named(self.ctx.handle, _abi.ptr(arr), _abi.ptr(buf), _abi.ptr(off), arr.shape[0], C.byref(h)),
                       self.ctx.handle)
        self.handle = h
        self._index = {p: i for i, p in enumerate(self.pks)}

    def close(self):
        if getattr(self, "handle", None):
            self._lib.afc_keyset_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def info(self):
        n, b = C.c_uint32(), C.c_uint64()
        _abi.check(self._lib.afc_keyset_info(self.handle, C.byref(n), C.byref(b)))
        return {"n_keys": n.value, "table_bytes": b.value}

    def index_of(self, pk):
        return self._index[bytes(pk)]

    def verify_packed(self, key_index, sigs, buf, off):
        n = len(off) - 1
        ki = np.ascontiguousarray(key_index, dtype=np.uint32)
        out = np.empty(n, dtype=np.uint8)
        _abi.check(self._lib.afc_ed25519_verify_keyed_batch(self.ctx.handle, self.handle, _abi.ptr(ki), _abi.ptr(sigs), _abi.ptr(buf), _abi.ptr(off),
                                                            n, _abi.ptr(out)), self.ctx.handle)
        return out

    def verify_dev(self, d_key_index, d_sigs, d_msgs, d_off, n, d_ok, stream=None):
        _abi.check(self._lib.afc_ed25519_verify_keyed_batch_dev(self.ctx.handle, self.handle, _abi.ptr(d_key_index), _abi.ptr(d_sigs), _abi.ptr(d_msgs),
                                                                _abi.ptr(d_off), n, _abi.ptr(d_ok), self.ctx._stream(stream)), self.ctx.handle)

    def verify_batch(self, pks, msgs, sigs):
        """VerifyBatch against registered issuers (same contract as Verifier.verify_batch)."""
        n = len(pks)
        if not (n == len(msgs) == len(sigs)):
            raise ValueError("pks, msgs and sigs must have the same length")
        if n == 0:
            return []
        ki = np.fromiter((self._index[bytes(p)] for p in pks), dtype=np.uint32, count=n)
        bad_len = [len(s) != 64 for s in sigs]
        sg = np.zeros((n, 64), dtype=np.uint8)
        for i, s in enumerate(sigs):
            if not bad_len[i]:
                sg[i] = np.frombuffer(s, dtype=np.uint8)
        buf, off = pack(msgs)
        ok = self.verify_packed(ki, sg, buf, off)
        return [bool(o) and not b for o, b in zip(ok, bad_len)]

    def verify_stored_packed(self, doc_kind, buf, off, fields=True):
        """afc_vc_verify_stored_batch: n stored documents (packed bytes + n+1 offsets) -> (status uint8 [n], fields uint32 [n, 4] or
        None).  doc_kind: _abi.DOC_EXECUTION_VC or _abi.DOC_WORKFLOW_VC; statuses are _abi.VC_*."""
        n = len(off) - 1
        st = np.empty(n, dtype=np.uint8)
        fl = np.empty((n, 4), dtype=np.uint32) if fields else None
        _abi.check(self._lib.afc_vc_verify_stored_batch(self.ctx.handle, self.handle, doc_kind, _abi.ptr(buf), _abi.ptr(off), n, _abi.ptr(st),
                                                        _abi.ptr(fl)), self.ctx.handle)
        return st, fl

    def verify_stored_dev(self, doc_kind, d_docs, d_off, n, d_status, d_fields=None, stream=None):
        _abi.check(self._lib.afc_vc_verify_stored_batch_dev(self.ctx.handle, self.handle, doc_kind, _abi.ptr(d_docs), _abi.ptr(d_off), n,
                                                            _abi.ptr(d_status), _abi.ptr(d_fields), self.ctx._stream(stream)), self.ctx.handle)

    def verify_stored(self, doc_kind, docs):
        """Host convenience: a list of stored documents (bytes) -> (statuses, fields)."""
        if not docs:
            return np.zeros(0, dtype=np.uint8), np.zeros((0, 4), dtype=np.uint32)
        buf, off = pack(docs)
        return self.verify_stored_packed(doc_kind, buf, off)

    def verify_json_packed(self, doc_kind, buf, off, fields=True):
        """afc_vc_verify_json_batch: verify_stored_packed for documents in any JSON spelling (request bodies, files), re-marshalled on
        the device.  Same statuses and fields (spans into each input document)."""
        n = len(off) - 1
        st = np.empty(n, dtype=np.uint8)
        fl = np.empty((n, 4), dtype=np.uint32) if fields else None
        _abi.check(self._lib.afc_vc_verify_json_batch(self.ctx.handle, self.handle, doc_kind, _abi.ptr(buf), _abi.ptr(off), n, _abi.ptr(st),
                                                      _abi.ptr(fl)), self.ctx.handle)
        return st, fl

    def verify_json_dev(self, doc_kind, d_docs, d_off, n, d_status, d_fields=None, stream=None):
        _abi.check(self._lib.afc_vc_verify_json_batch_dev(self.ctx.handle, self.handle, doc_kind, _abi.ptr(d_docs), _abi.ptr(d_off), n,
                                                          _abi.ptr(d_status), _abi.ptr(d_fields), self.ctx._stream(stream)), self.ctx.handle)

    def verify_json(self, doc_kind, docs):
        """Host convenience: a list of documents in any JSON spelling (bytes) -> (statuses, fields)."""
        if not docs:
            return np.zeros(0, dtype=np.uint8), np.zeros((0, 4), dtype=np.uint32)
        buf, off = pack(docs)
        return self.verify_json_packed(doc_kind, buf, off)

    def verify_requests_packed(self, reqs, req_off):
        """afc_vc_verify_request_batch: n raw request bodies of POST /api/v1/did/verify (packed bytes + n+1 offsets) -> (bodies uint8,
        body_off uint64 [n+1], state uint8 [n] of _abi.VREQ_*)."""
        n = len(req_off) - 1
        cap = self._lib.afc_vc_verify_request_bound(_abi.ptr(req_off), n)
        bodies = np.empty(max(cap, 1), dtype=np.uint8)
        body_off = np.zeros(n + 1, dtype=np.uint64)
        state = np.empty(max(n, 1), dtype=np.uint8)
        _abi.check(self._lib.afc_vc_verify_request_batch(self.ctx.handle, self.handle, _abi.ptr(reqs), _abi.ptr(req_off), n, _abi.ptr(bodies), cap,
                                                         _abi.ptr(body_off), _abi.ptr(state)), self.ctx.handle)
        return bodies[:int(body_off[n])], body_off, state[:n]

    def verify_requests_dev(self, d_reqs, d_req_off, n, stream=None):
        """afc_vc_verify_request_batch_dev on device tensors (request bytes uint8, offsets int64 [n+1]).  Returns (d_bodies uint8,
        d_body_off int64 [n+1], d_state uint8 [n])."""
        import torch
        dev = d_req_off.device
        cap = 0
        if n:
            a, b = (int(x) for x in torch.cat([d_req_off[0:1], d_req_off[n:n + 1]]).cpu().tolist())
            cap = self._lib.afc_vc_verify_request_bound(_abi.ptr(np.array([a, max(a, b)], dtype=np.uint64)), 1) + \
                (n - 1) * self._lib.afc_vc_verify_request_bound(_abi.ptr(np.zeros(2, dtype=np.uint64)), 1)
        d_bodies = torch.empty(max(cap, 1), dtype=torch.uint8, device=dev)
        d_body_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_state = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
        _abi.check(self._lib.afc_vc_verify_request_batch_dev(self.ctx.handle, self.handle, _abi.ptr(d_reqs), _abi.ptr(d_req_off), n, _abi.ptr(d_bodies),
                                                             cap, _abi.ptr(d_body_off), _abi.ptr(d_state), self.ctx._stream(stream)), self.ctx.handle)
        total = int(d_body_off[n]) if n else 0
        return d_bodies[:total], d_body_off, d_state[:n]

    def verify_requests(self, bodies):
        """Many request bodies (bytes) in one host-buffer call: [(state, response body bytes)] in request order (an _abi.VREQ_HOST request
        has an empty body)."""
        if not bodies:
            return []
        buf, off = pack([bytes(b) for b in bodies])
        out, body_off, state = self.verify_requests_packed(buf, off)
        raw = out.tobytes()
        return [(int(state[i]), raw[int(body_off[i]):int(body_off[i + 1])]) for i in range(len(bodies))]

    def audit_stored_packed(self, doc_kind, buf, off, cols=None, col_off=None):
        """afc_vc_audit_stored_batch: n stored documents (packed bytes + n+1 offsets) and, for execution documents, their records'
        _abi.AUDIT_COLUMNS columns (packed bytes + n*10+1 offsets) -> (status uint8 [n], issues uint32 [n] of _abi.AUDIT_* bits)."""
        n = len(off) - 1
        st = np.empty(n, dtype=np.uint8)
        iss = np.empty(n, dtype=np.uint32)
        _abi.check(self._lib.afc_vc_audit_stored_batch(self.ctx.handle, self.handle, doc_kind, _abi.ptr(buf), _abi.ptr(off), _abi.ptr(cols),
                                                       _abi.ptr(col_off), n, _abi.ptr(st), _abi.ptr(iss)), self.ctx.handle)
        return st, iss

    def audit_stored_dev(self, doc_kind, d_docs, d_off, d_cols, d_col_off, n, d_status, d_issues, stream=None):
        _abi.check(self._lib.afc_vc_audit_stored_batch_dev(self.ctx.handle, self.handle, doc_kind, _abi.ptr(d_docs), _abi.ptr(d_off), _abi.ptr(d_cols),
                                                           _abi.ptr(d_col_off), n, _abi.ptr(d_status), _abi.ptr(d_issues), self.ctx._stream(stream)),
                   self.ctx.handle)

    def audit_stored(self, doc_kind, docs, columns=None):
        """Host convenience: stored documents (bytes) and, for execution documents, one sequence of _abi.AUDIT_COLUMNS values (str or
        bytes; str is encoded as UTF-8, lone surrogates kept as their three bytes) per document -> (statuses, issue masks)."""
        if not docs:
            return np.zeros(0, dtype=np.uint8), np.zeros(0, dtype=np.uint32)
        buf, off = pack(docs)
        if columns is None:
            return self.audit_stored_packed(doc_kind, buf, off)
        if len(columns) != len(docs) or any(len(c) != len(_abi.AUDIT_COLUMNS) for c in columns):
            raise ValueError("one row of %d columns per document" % len(_abi.AUDIT_COLUMNS))
        flat = [v.encode("utf-8", "surrogatepass") if isinstance(v, str) else bytes(v) for row in columns for v in row]
        cbuf, coff = pack(flat)
        return self.audit_stored_packed(doc_kind, buf, off, cbuf, coff)
