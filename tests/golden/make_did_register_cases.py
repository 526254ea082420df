"""Writes tests/golden/did_register_cases.json: agent DID registrations (handleNewRegistration) through oracle/ref_did.py for a fixed
master seed and server id — an agent with no components, empty ids, duplicates, every escape class, invalid UTF-8, non-ASCII ids in raw
byte order, long ids.  Byte strings are hex; each component's seed is pinned by its SHA-256 only.

    python tests/golden/make_did_register_cases.py
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import did_cases as DC  # noqa: E402

AGENT_BASE = 7


def main():
    reqs = DC.golden_requests()
    cases = []
    for r, w in zip(reqs, DC.oracle(reqs, AGENT_BASE)):
        cases.append({"agent_node_id": r["agent_node_id"].hex(), "reasoners": [x.hex() for x in r["reasoners"]],
                      "skills": [x.hex() for x in r["skills"]], "body": w["body"].hex(),
                      "components": [{"path": c["path"].decode(), "did": c["did"].decode(), "pk": c["pk"].hex(),
                                      "seed_sha256": hashlib.sha256(c["seed"]).hexdigest(), "kept": c["kept"]} for c in w["components"]]})
    doc = {"master_seed": DC.MASTER.hex(), "server_id": DC.SERVER.hex(), "agent_base": AGENT_BASE, "cases": cases}
    with open(os.path.join(HERE, "did_register_cases.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
