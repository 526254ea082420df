"""Workflow-credential cases shared by the CPU and GPU tests of afc_vc_issue_workflow_batch, and what the oracle says about them.

A case is {"cols": [7 byte strings in AFC_WORKFLOW_COLUMNS order], "records": [(vc_id bytes, status bytes, seconds, nanoseconds), ...]}.
The expectations come from oracle/ref_vc.py (workflow_vc_document, go_marshal, determine_workflow_status), Python's datetime for the
RFC 3339 text, and the plain Go rules for the start / end records (the first strict minimum and maximum)."""
import datetime as dt

import numpy as np

from oracle import ref_vc as RV

COLUMNS = ("workflow_id", "session_id", "issuer_did", "vc_id", "issuance_date", "snapshot_time", "proof_created")
STATUS_IDS = {"unknown": 0, "pending": 1, "queued": 2, "running": 3, "succeeded": 4, "failed": 5, "cancelled": 6, "timeout": 7}
# every name NormalizeExecutionStatus knows (pkg/types/status.go:28-63): the eight canonical ones and the sixteen aliases
STATUS_SPELLINGS = ("unknown", "pending", "queued", "running", "succeeded", "failed", "cancelled", "timeout", "success", "successful", "completed",
                    "complete", "done", "ok", "error", "failure", "errored", "canceled", "cancel", "timed_out", "wait", "waiting", "in_progress",
                    "processing")
SEC_MIN, SEC_MAX = -62135596800, 253402300799                # 0001-01-01T00:00:00Z, 9999-12-31T23:59:59Z
NONE = 0xFFFFFFFF
PLACEHOLDER = "A" * 86
# strings of every escape class json.Marshal has, and invalid UTF-8 (a lone continuation byte, a cut rune, an overlong form, a surrogate)
ODD = [b'q"uote', b"back\\slash", b"ctl\x00\x01\x1f\x7f", b"<html>&amp;", "line\u2028sep".encode(), "para\u2029sep".encode(),
       "é中\U0001F600".encode(), b"", b"tab\there\n\r\b\f", b"bad\x80byte", b"cut\xe4\xb8", b"over\xc0\xaf", b"sur\xed\xa0\x80"]


def normalize(status: bytes) -> str:
    """NormalizeExecutionStatus of a status the device decides (printable ASCII and \\t \\n \\v \\f \\r)."""
    s = status.decode("ascii").strip(" \t\n\v\f\r").lower()
    if s in STATUS_IDS:
        return s
    alias = {"success": "succeeded", "successful": "succeeded", "completed": "succeeded", "complete": "succeeded", "done": "succeeded",
             "ok": "succeeded", "error": "failed", "failure": "failed", "errored": "failed", "canceled": "cancelled", "cancel": "cancelled",
             "timed_out": "timeout", "wait": "queued", "waiting": "queued", "in_progress": "running", "processing": "running"}
    return alias.get(s, "unknown")


def decided(status: bytes) -> bool:
    return all(0x20 <= c <= 0x7E or c in b"\t\n\v\f\r" for c in status)


def is_host(case) -> bool:
    return any(not decided(st) or not SEC_MIN <= s <= SEC_MAX or not 0 <= ns < 10 ** 9 for _, st, s, ns in case["records"])


def time_text(sec: int) -> str:
    t = dt.datetime(1970, 1, 1) + dt.timedelta(seconds=sec)
    return "%04d-%02d-%02dT%02d:%02d:%02dZ" % (t.year, t.month, t.day, t.hour, t.minute, t.second)


def summary(case):
    """[status id, completed, start, end] as the call reports it, or None for a HOST workflow."""
    if is_host(case):
        return None
    recs = case["records"]
    if not recs:
        return [STATUS_IDS["pending"], 0, NONE, NONE]
    names = [normalize(st) for _, st, _, _ in recs]
    status = RV.determine_workflow_status(names)
    keys = [(s, ns) for _, _, s, ns in recs]
    start = keys.index(min(keys))
    end = keys.index(max(keys)) if status in ("succeeded", "failed", "cancelled", "timeout") else NONE
    return [STATUS_IDS[status], names.count("succeeded"), start, end]


def go_str(raw: bytes) -> str:
    return RV._go_bytes_as_str(raw)


def oracle_docs(case, proof_value=PLACEHOLDER):
    """(signing message, stored document) of a built workflow from oracle/ref_vc.py."""
    c = {k: go_str(v) for k, v in zip(COLUMNS, case["cols"])}
    s = summary(case)
    recs = case["records"]
    w = {"workflow_id": c["workflow_id"], "session_id": c["session_id"], "component_vc_ids": [go_str(r[0]) for r in recs],
         "status": [k for k, v in STATUS_IDS.items() if v == s[0]][0],
         "start_time": time_text(recs[s[2]][2]) if recs else c["snapshot_time"],
         "end_time": time_text(recs[s[3]][2]) if s[3] != NONE else None, "snapshot_time": c["snapshot_time"], "issuer_did": c["issuer_did"],
         "vc_id": c["vc_id"], "issuance_date": c["issuance_date"], "proof_created": c["proof_created"]}
    proof = {"type": "Ed25519Signature2020", "created": c["proof_created"], "verificationMethod": "%s#key-1" % c["issuer_did"],
             "proofPurpose": "assertionMethod", "proofValue": proof_value}
    return RV.go_marshal(RV.workflow_vc_document(w)), RV.go_marshal(RV.workflow_vc_document(w, proof))


def pack(cases):
    """The packed inputs of afc_vc_issue_workflow_batch: cols, col_off, rec_off, rec_cols, rec_col_off, created_at."""
    flat = [v for c in cases for v in c["cols"]]
    recs = [r for c in cases for r in c["records"]]
    rflat = [v for r in recs for v in (r[0], r[1])]

    def packed(vals):
        off = np.zeros(len(vals) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(v) for v in vals], dtype=np.uint64)
        return np.frombuffer(b"".join(vals) + b"\0" * 8, dtype=np.uint8).copy(), off
    cols, col_off = packed(flat)
    rec_cols, rec_col_off = packed(rflat)
    rec_off = np.zeros(len(cases) + 1, dtype=np.uint64)
    rec_off[1:] = np.cumsum([len(c["records"]) for c in cases], dtype=np.uint64)
    created = np.array([x for r in recs for x in (r[2], r[3])], dtype=np.int64).reshape(-1)
    return cols, col_off, rec_off, rec_cols, rec_col_off, created


def base_cols(i=0, issuer=b"did:key:z7QEA-r41xWlBHtUwbuCfQcjpzigXxQ7kGf2zKSPFlF4v_A"):
    return [b"wf_%04d" % i, b"sess_%04d" % i, issuer, b"vc-17%015d" % i, b"2026-09-21T06:00:00Z", b"2026-09-21T06:00:05Z", b"2026-09-21T06:00:06Z"]


def random_case(rng, i, issuer, max_records=12, odd=0.0, spellings=STATUS_SPELLINGS, t0=1_790_000_000):
    """A workflow with 0..max_records records, statuses from `spellings` with case and whitespace variants, ids shaped like generateVCID's
    vc-<nanos>, times in a small window (ties happen); with probability `odd` a column or id gets a string of ODD appended."""
    cols = base_cols(i, issuer)
    for k in range(7):
        if k != 2 and rng.random() < odd:
            cols[k] = cols[k] + ODD[int(rng.integers(len(ODD)))]
    recs = []
    for j in range(int(rng.integers(0, max_records + 1))):
        st = spellings[int(rng.integers(len(spellings)))].encode()
        v = int(rng.integers(4))
        st = st.upper() if v == 1 else st.title() if v == 2 else b" \t" + st + b"\n" if v == 3 else st
        vid = b"vc-%d" % (1_790_000_000_000_000_000 + 1000 * i + j)
        if rng.random() < odd:
            vid = vid + ODD[int(rng.integers(len(ODD)))]
        recs.append((vid, st, t0 + int(rng.integers(0, 40)), int(rng.choice([0, 999_999_999, int(rng.integers(10 ** 9))]))))
    return {"cols": cols, "records": recs}


def oracle_signed(case, seed: bytes):
    """(stored document, proofValue) of a built workflow, signed by OpenSSL over the oracle's signing message."""
    import base64
    from cryptography.hazmat.primitives.asymmetric.ed25519 import Ed25519PrivateKey
    msg, _ = oracle_docs(case)
    pv = base64.urlsafe_b64encode(Ed25519PrivateKey.from_private_bytes(seed).sign(msg)).rstrip(b"=").decode()
    return oracle_docs(case, pv)[1], pv


def bulk(n, rng, issuers, max_records=32, skew=None, counts=None):
    """n workflows as packed arrays without Python objects per record (for the large runs): each has 0..max_records records (with `skew` =
    (fraction, count): that fraction of the workflows has `count` records; `counts`: each workflow's count), ids vc-<19 digits>, statuses from a realistic mix, times in a
    window of an hour.  Returns (key_index, cols, col_off, rec_off, rec_cols, rec_col_off, created_at) and a function that rebuilds case i."""
    counts = rng.integers(0, max_records + 1, n) if counts is None else np.array(counts)
    if skew is not None:
        counts[rng.random(n) < skew[0]] = skew[1]
    rec_off = np.zeros(n + 1, dtype=np.uint64)
    rec_off[1:] = np.cumsum(counts, dtype=np.uint64)
    m = int(rec_off[n])
    mix = [b"succeeded", b"completed", b"failed", b"running", b"cancelled", b"timeout", b"queued", b"pending", b"SUCCESS", b" done "]
    p = np.array([0.55, 0.15, 0.06, 0.08, 0.03, 0.02, 0.04, 0.03, 0.02, 0.02])
    st = rng.choice(len(mix), m, p=p)
    # every workflow has one issuer; a workflow whose records all succeeded is the common case
    ki = rng.integers(0, len(issuers), n).astype(np.uint32)
    idw = 22
    ids = np.frombuffer(b"".join(b"vc-%019d" % (1_790_000_000_000_000_000 + r) for r in range(m)), dtype=np.uint8).reshape(m, idw) if m else \
        np.zeros((0, idw), dtype=np.uint8)
    slen = np.array([len(s) for s in mix])[st]
    rec_col_off = np.zeros(2 * m + 1, dtype=np.uint64)
    lens = np.empty(2 * m, dtype=np.uint64)
    lens[0::2] = idw
    lens[1::2] = slen
    rec_col_off[1:] = np.cumsum(lens, dtype=np.uint64)
    rec_cols = np.empty(int(rec_col_off[-1]) + 8, dtype=np.uint8)
    starts = rec_col_off[0:-1:2].astype(np.int64)
    for k in range(idw):
        rec_cols[starts + k] = ids[:, k]
    sstart = rec_col_off[1::2].astype(np.int64)
    for j, s in enumerate(mix):
        sel = sstart[st == j]
        for k, c in enumerate(s):
            rec_cols[sel + k] = c
    created = np.empty(2 * m, dtype=np.int64)
    created[0::2] = 1_790_000_000 + rng.integers(0, 3600, m)
    created[1::2] = rng.integers(0, 10 ** 9, m)
    cols_list = []
    for i in range(n):
        cols_list += [b"wf_%08d" % i, b"sess_%08d" % i, issuers[ki[i]].encode(), b"%d" % (1_790_000_000_000_000_000 + i), b"2026-09-21T06:00:00Z",
                      b"2026-09-21T06:00:05Z", b"2026-09-21T06:00:06Z"]
    col_off = np.zeros(7 * n + 1, dtype=np.uint64)
    col_off[1:] = np.cumsum([len(v) for v in cols_list], dtype=np.uint64)
    cols = np.frombuffer(b"".join(cols_list) + b"\0" * 8, dtype=np.uint8).copy()

    def case(i):
        a, b = int(rec_off[i]), int(rec_off[i + 1])
        recs = []
        for r in range(a, b):
            o = [int(x) for x in rec_col_off[2 * r:2 * r + 3]]
            recs.append((rec_cols[o[0]:o[1]].tobytes(), rec_cols[o[1]:o[2]].tobytes(), int(created[2 * r]), int(created[2 * r + 1])))
        return {"cols": cols_list[7 * i:7 * i + 7], "records": recs}
    return (ki, cols, col_off, rec_off, rec_cols, rec_col_off, created), case
