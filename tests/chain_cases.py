"""Workflow-chain cases shared by the CPU and GPU tests of afc_vc_workflow_chain_batch: the golden fixture's cases, seeded random
workflows, a directory, and the packed arrays of the call.  Expectations come from tests/chain_oracle.py."""
import json
import os

import numpy as np

import chain_oracle as CO
import workflow_cases as WC

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "workflow_chain_cases.json")
T0 = 1_790_000_000


def pk_of(did: bytes) -> bytes:
    import hashlib
    return hashlib.sha256(b"pk:" + did).digest()


def record(vc_id, status=b"succeeded", sec=T0, nsec=0, zone=0, issuer=b"did:key:zIssuer", caller=b"did:key:zCaller", target=b"did:key:zTarget",
           doc=b'{"a":1}', flags=0, agent=b"agent-1", name=b"wf-name", doc_size=None):
    cols = [b"exec-" + vc_id, b"wf-1", b"sess-1", agent, name, issuer, target, caller, doc, b"sig-" + vc_id, b"", b"in-hash", b"out-hash"]
    return {"vc_id": vc_id, "status": status, "sec": sec, "nsec": nsec, "zone": zone, "cols": cols, "flags": flags,
            "doc_size": len(doc) if doc_size is None else doc_size}


def workflow(i, records, issuer=b"did:key:zIssuer", clock=(T0 + 100, 5, 0), resolved_at=b"2026-09-21T06:00:07Z"):
    cols = WC.base_cols(i, issuer)
    if records:
        cols[1] = records[0]["cols"][2]
    return {"cols": cols, "records": records, "wf_vc_id": b"vc-wf-%d" % i, "resolved_at": resolved_at, "clock": clock}


DIRECTORY_DIDS = [b"did:key:zIssuer", b"did:key:zCaller", b"did:key:zTarget", b"did:web:example.com:agent", b"did:", b"did::x", b"did:key:",
                  "did:key:　".encode(), b"did:key:z<esc>&\"q\"", b"did:key:z\x7f", b"did:key:zA", b"did:key:z\xe2\x80\xa8", b"did:key:z~",
                  b"plain-name", b"did:key:zB\\", "did:key:zé".encode(), b"did:web:" + b"x" * 121]


def directory(extra=()):
    dids = list(DIRECTORY_DIDS) + list(extra)
    return {d: pk_of(d) for d in dids}


def fixture_cases():
    """The fixture's workflows: every rule the body depends on."""
    R = record
    cases = [
        workflow(0, []),                                                                     # no records; the issuer alone in the bundle
        workflow(1, [R(b"vc-1", flags=CO.AGENT_NIL | CO.NAME_NIL), R(b"vc-2", agent=b"", name=b"", sec=T0 + 1)]),   # nil vs empty
        workflow(2, [R(b"vc-1", flags=CO.DOC_NIL), R(b"vc-2", doc=b' { "k" : [1, 2,\n\t3 ] ,"s":"a b"}\r\n', sec=T0 + 2),
                     R(b"vc-3", doc='{"h":"<b>&amp;</b>","ls":"x y "}'.encode(), sec=T0 + 3),
                     R(b"vc-4", doc=b'"\\u003c\\"<"', status=b"failed")]),                     # nil, indented, HTML characters
        workflow(3, [R(b"vc-1", doc=b"")]),                                                   # non-nil empty document: HOST
        workflow(4, [R(b"vc-1", doc=b'{"a":}')]),                                             # invalid document: HOST
        workflow(5, [R(b"vc-1", zone=0, nsec=0), R(b"vc-2", zone=19800, nsec=500_000_000, sec=T0 + 5),
                     R(b"vc-3", zone=-28800, nsec=1, sec=T0 + 9, status=b"done")], clock=(T0 + 50, 123_456_789, 19800)),
        workflow(6, [R(b"vc-1", zone=19830)]),                                                 # an offset with seconds: HOST
        workflow(7, [R(b"vc-1", issuer=b"", caller=b"did:key:", target=b" \t\n"), R(b"vc-2", issuer="　".encode(), caller=b"did:key:zUnknown",
                                                                                        target=b"did:key:zTarget")], issuer=b"did:key:zIssuer"),
        workflow(8, [R(b"vc-1", issuer=b"did:", caller=b"did::x", target=b"did:web:example.com:agent"),
                     R(b"vc-2", issuer=b"did:key:z<esc>&\"q\"", caller=b"did:key:z\x7f", target=b"did:key:zA"),
                     R(b"vc-3", issuer="did:key:zé".encode(), caller=b"did:key:z\xe2\x80\xa8", target=b"did:key:z~"),
                     R(b"vc-4", issuer=b"plain-name", caller=b"did:key:zB\\", target=b"did:key:zA")], issuer=b"did:key:zA"),
        workflow(9, [R(b"vc-1", issuer=b"did:key:zNone", caller=b"", target=b"")], issuer=b"did:key:zNope"),   # empty bundle: omitted
        workflow(10, [R(b"vc-1", status=b"succ\x01eeded")]),                                  # the issue passes decline it: HOST
        workflow(11, [R(b"vc-%d" % k, sec=T0 + k % 3, nsec=k, status=b"completed") for k in range(40)]),
        workflow(12, [R(b"vc-1")], issuer=b""),                                               # no issuer_did member
        workflow(13, [R(b"vc-1")], resolved_at=b"x" * 65),                                    # resolved_at too long: HOST
        workflow(14, [R(b"vc-1", target=b"did:web:" + b"x" * 121)]),                          # a bundle DID of 129 bytes: HOST
        workflow(15, [R(b"vc-1", target=b"did:web:" + b"x" * 120)]),                          # 128 bytes: built
    ]
    return cases


def random_case(rng, i, dids):
    """A workflow of 0..12 records over a pool of DIDs (some outside the directory), random documents, zones and nanoseconds."""
    docs = [b'{"a":1}', b' [1, {"b" : "<x>"} ]', b'"s"', b"null", b'{"k":"\\u2028 \xe2\x80\xa8 &"}', b"{", b"", b"  7  "]
    zones = [0, 0, 3600, -18000, 19800, 20700, -34200, 50400, 45]
    recs = []
    for k in range(int(rng.integers(0, 13))):
        pick = lambda: dids[int(rng.integers(len(dids)))]
        flags = int(rng.integers(8)) if rng.random() < 0.3 else 0
        st = WC.STATUS_SPELLINGS[int(rng.integers(len(WC.STATUS_SPELLINGS)))].encode()
        recs.append(record(b"vc-%d-%d" % (i, k), status=st, sec=T0 + int(rng.integers(0, 40)), nsec=int(rng.choice([0, 1, 500_000_000, int(rng.integers(10 ** 9))])),
                           zone=int(rng.choice(zones)) if rng.random() < 0.98 else 30, issuer=pick(), caller=pick(), target=pick(),
                           doc=docs[int(rng.integers(len(docs)))] if rng.random() < 0.9 else docs[0], flags=flags,
                           agent=b"" if rng.random() < 0.2 else b"agent-%d" % k, doc_size=int(rng.integers(0, 10 ** 6))))
    return workflow(i, recs, issuer=dids[int(rng.integers(len(dids)))], clock=(T0 + 100, int(rng.integers(10 ** 9)), int(rng.choice(zones[:8]))))


def random_dids(extra=24):
    return list(DIRECTORY_DIDS) + [b"did:key:zR%03d" % k for k in range(extra)] + [b"did:key:zMissing%d" % k for k in range(6)] + [b"", b" "]


def pack(cases):
    """The host arrays of afc_vc_workflow_chain_batch after key_index: (issue arrays..., chain_cols, chain_col_off, clock, chain_rec_cols,
    chain_rec_col_off, rec_flags, doc_size, created_off)."""
    cols, col_off, rec_off, rec_cols, rec_col_off, created = WC.pack([CO.issue_case(c) for c in cases])

    def packed(vals):
        off = np.zeros(len(vals) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(v) for v in vals], dtype=np.uint64)
        return np.frombuffer(b"".join(vals) + b"\0" * 8, dtype=np.uint8).copy(), off
    chain_cols, chain_col_off = packed([v for c in cases for v in (c["wf_vc_id"], c["resolved_at"])])
    recs = [r for c in cases for r in c["records"]]
    chain_rec_cols, chain_rec_col_off = packed([v for r in recs for v in r["cols"]])
    clock = np.array([x for c in cases for x in c["clock"]], dtype=np.int64)
    flags = np.array([r["flags"] for r in recs] + [0], dtype=np.uint8)
    size = np.array([r["doc_size"] for r in recs] + [0], dtype=np.int64)
    zone = np.array([r["zone"] for r in recs] + [0], dtype=np.int32)
    created = np.ascontiguousarray(created if len(created) else np.zeros(2, dtype=np.int64))
    return (cols, col_off, rec_off, rec_cols, rec_col_off, created, chain_cols, chain_col_off, clock, chain_rec_cols, chain_rec_col_off, flags, size,
            zone)


def pack_directory(d):
    dids = list(d)
    buf = np.frombuffer(b"".join(dids) + b"\0" * 8, dtype=np.uint8).copy()
    off = np.zeros(len(dids) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(x) for x in dids], dtype=np.uint64)
    pks = np.frombuffer(b"".join(d[x] for x in dids) or b"\0" * 32, dtype=np.uint8).copy()
    return pks, buf, off


def _hex(b):
    return b.hex()


def to_json(cases):
    out = []
    for c in cases:
        out.append({"cols": [_hex(v) for v in c["cols"]], "wf_vc_id": _hex(c["wf_vc_id"]), "resolved_at": _hex(c["resolved_at"]), "clock": list(c["clock"]),
                    "records": [dict(r, vc_id=_hex(r["vc_id"]), status=_hex(r["status"]), cols=[_hex(v) for v in r["cols"]]) for r in c["records"]]})
    return out


def from_json(items):
    cases = []
    for c in items:
        cases.append({"cols": [bytes.fromhex(v) for v in c["cols"]], "wf_vc_id": bytes.fromhex(c["wf_vc_id"]), "resolved_at": bytes.fromhex(c["resolved_at"]),
                      "clock": tuple(c["clock"]), "records": [dict(r, vc_id=bytes.fromhex(r["vc_id"]), status=bytes.fromhex(r["status"]),
                                                                    cols=[bytes.fromhex(v) for v in r["cols"]]) for r in c["records"]]})
    return cases


def load_fixture():
    """(cases, directory, expected [(state, body with the placeholder proof value)])."""
    with open(FIXTURE) as f:
        fx = json.load(f)
    d = {bytes.fromhex(k): bytes.fromhex(v) for k, v in fx["directory"]}
    return from_json(fx["cases"]), d, [(e["state"], bytes.fromhex(e["body"])) for e in fx["expected"]]
