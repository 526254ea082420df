"""Writes tests/golden/did_reregister_cases.json: known-agent re-registrations (RegisterAgent's branch for an agent the registry holds)
through the oracle of tests/didrr_oracle.py for a fixed master seed and server id: every state, repeated new ids, the shared path index
(also a new reasoner that receives a surviving component's DID after a removal), empty ids and lists, ids and columns that need
escaping, a stored JWK in a non-canonical spelling, an empty stored function_name.  Byte strings are hex; each key slot's seed is pinned
by its SHA-256 only.

    python tests/golden/make_did_reregister_cases.py
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import didrr_cases as RC  # noqa: E402


def main():
    reqs = RC.golden_requests()
    cases = []
    for r, w in zip(reqs, RC.oracle(reqs)):
        slots = [None if s is None else {"path": s["path"].decode(), "did": s["did"].decode(), "pk": s["pk"].hex(),
                                         "seed_sha256": hashlib.sha256(s["seed"]).hexdigest()} for s in w["slots"]]
        cases.append({"request": RC.to_json(r), "state": w["state"], "counts": w["counts"], "body": w["body"].hex(), "gone": w["gone"],
                      "id_flags": w["id_flags"], "slots": slots})
    doc = {"master_seed": RC.MASTER.hex(), "server_id": RC.SERVER.hex(), "cases": cases}
    with open(os.path.join(HERE, "did_reregister_cases.json"), "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
