"""Writes tests/golden/workflow_chain_cases.json: the workflow-chain cases of tests/chain_cases.py, the directory they resolve against,
and each case's state and body (signed with the placeholder proof value) as tests/chain_oracle.py computes them.

    python tests/golden/make_workflow_chain_cases.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import chain_cases as CC  # noqa: E402
import chain_oracle as CO  # noqa: E402


def main():
    cases, d = CC.fixture_cases(), CC.directory()
    expected = []
    for c in cases:
        host = CO.is_host(c, d)
        expected.append({"state": 1 if host else 0, "body": "" if host else CO.chain_body(c, d).hex()})
    with open(CC.FIXTURE, "w") as f:
        json.dump({"directory": [[k.hex(), v.hex()] for k, v in d.items()], "cases": CC.to_json(cases), "expected": expected}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
