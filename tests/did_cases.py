"""Agent DID registration cases shared by the CPU and GPU tests and the fixture generator: requests as afc_did_register_batch packs
them, and what oracle/ref_did.py says the reference returns for them."""
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_did as RD  # noqa: E402

MASTER = bytes(range(0x40, 0x60))
SERVER = b"agentfield-server-01"

ESCAPES = [b"a\"b", b"back\\slash", b"<tag>&amp", b"ctl\x01\x1f\x7f", b"nl\n\r\t\b\x0c", b"sep\xe2\x80\xa8\xe2\x80\xa9", b"bad\xff\xfe",
           b"cut\xe2\x82", b"\xc3\xa9t\xc3\xa9", b"\xf0\x9f\x98\x80emoji", b"\xed\xa0\x80surrogate", b"\xc0\xafoverlong"]


def pack(requests):
    """requests: dicts of bytes agent_node_id, reasoners, skills -> (nodes, node_off, id_idx, ids, id_off) as uint8 / uint64 arrays."""
    def cat(xs):
        off = np.zeros(len(xs) + 1, dtype=np.uint64)
        if xs:
            off[1:] = np.cumsum([len(x) for x in xs])
        buf = np.frombuffer(b"".join(xs) + b"\0", dtype=np.uint8).copy()
        return buf, off
    flat, idx = [], [0]
    for r in requests:
        flat += list(r["reasoners"])
        idx.append(len(flat))
        flat += list(r["skills"])
        idx.append(len(flat))
    nodes, node_off = cat([r["agent_node_id"] for r in requests])
    ids, id_off = cat(flat)
    return nodes, node_off, np.array(idx, dtype=np.uint64), ids, id_off


def oracle(requests, agent_base=0, master=MASTER, server=SERVER):
    return [RD.register(master, server, r["agent_node_id"], r["reasoners"], r["skills"], agent_base + k) for k, r in enumerate(requests)]


def random_requests(rng: random.Random, n, max_ids=8, dup=0.2, esc=0.1, empty=0.05, alphabet=4):
    """Requests with heavily repeated ids (drawn from a small pool), some empty and some that need escaping."""
    pool = [b"fn_%d" % k for k in range(alphabet)] + [b"fn_%d_x" % k for k in range(alphabet)]

    def one():
        u = rng.random()
        if u < empty:
            return b""
        if u < empty + esc:
            return rng.choice(ESCAPES) + (b"%d" % rng.randrange(3))
        if u < empty + esc + dup:
            return rng.choice(pool)
        return b"summarize_text_%d" % rng.randrange(10 ** rng.randrange(1, 8))
    out = []
    for i in range(n):
        node = b"node-%d" % i if rng.random() > esc else rng.choice(ESCAPES) + b"-%d" % i
        out.append({"agent_node_id": node, "reasoners": [one() for _ in range(rng.randrange(max_ids + 1))],
                    "skills": [one() for _ in range(rng.randrange(max_ids + 1))]})
    return out


def golden_requests():
    """The fixture's requests: an agent with no components; empty ids; duplicates; every escape class; invalid UTF-8; non-ASCII ids
    (raw byte order is not code point order for U+FFFF vs U+10000); long ids (two-block hashes and one-block ones)."""
    return [
        {"agent_node_id": b"bare-agent", "reasoners": [], "skills": []},
        {"agent_node_id": b"empties", "reasoners": [b"", b"r1", b"", b"r2"], "skills": [b"", b""]},
        {"agent_node_id": b"dups", "reasoners": [b"a", b"b", b"a", b"c", b"b", b"a"], "skills": [b"s", b"s"]},
        {"agent_node_id": b"esc<&>\"\\\n", "reasoners": ESCAPES[:6], "skills": ESCAPES[6:]},
        {"agent_node_id": b"bad\xff\xc3", "reasoners": [b"\xff", b"\xfe\xff", b"ok"], "skills": [b"\xe2\x80"]},
        {"agent_node_id": b"unicode", "reasoners": [b"\xef\xbf\xbd", b"\xf0\x90\x80\x80", b"z", b"\xc3\xa9", b"e\xcc\x81", b"Z"],
         "skills": [b"\xe4\xb8\xad\xe6\x96\x87", b"\xe6\x97\xa5\xe6\x9c\xac"]},
        {"agent_node_id": b"summarizer", "reasoners": [b"summarize_text_%d" % k for k in range(12)], "skills": [b"tag_%d" % k for k in range(11)]},
    ]
