"""Writes tests/golden/did_resolve_cases.json: the registry and requests of tests/resolve_cases.py and, per request, every outcome
tests/resolve_oracle.py allows ((status, body, host_ok); long requests and bodies in the compact forms resolve_cases describes).

    python tests/golden/make_did_resolve_cases.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import resolve_cases as RC  # noqa: E402
import resolve_oracle as RO  # noqa: E402


def main():
    reg = RC.fixture_registry()
    reqs = RC.fixture_requests(reg)
    with open(RC.FIXTURE, "w") as f:
        json.dump({"registry": RC.registry_to_json(reg), "requests": [RC.request_json(k, d) for k, d in reqs],
                   "expected": [RC.outcomes_json(RO.outcomes(reg, k, d)) for k, d in reqs]}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
