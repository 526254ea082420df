"""Writes tests/golden/verify_request_cases.json: request bodies of POST /api/v1/did/verify around the golden execution credentials (every
response row, the envelope and syntax cases, the verdict variants) with the status and body tests/verify_request_oracle.py gives each.
baseline/go/gen_golden_test.go pins the same cases against gin's binding and VerifyVC where Go 1.24 runs.

    python tests/golden/make_verify_request_cases.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import test_vcreq_gpu as G  # noqa: E402
import test_vcreq_hostsim as H  # noqa: E402
import verify_request_oracle as O  # noqa: E402


def bodies():
    docs = H.realistic_docs()
    out = [shape(docs[0]) for shape in H.SHAPES]
    for v in G._variants(docs[1]):
        out.append(b'{"vc_document":' + v + b'}')
    doc = docs[2]
    out += [b'{"a":1,"vc_document":' + doc + b',"z":[{}]}', b'{"VC_DOCUMENT":' + doc + b'}', b'{"vc_document":' + doc + b'} x',
            b'{"vc_document":' + docs[3] + b',"vc_document":' + doc + b'}', b'{"vc_document":' + doc + b',"vc_document":null}',
            b'\xef\xbb\xbf{}', b'', b' ', b'[]', b'"x"', b'1', b'true', b'null', b'{}', b'{"vc_document":null}', b'{"vc_document":"x"}',
            b'{"vc_document":[]}', b'{"vc_document":-1e5}', b'{"vc_document":false}', b'{"vc_\\u0064ocument":' + doc + b'}',
            b'{"vc_document":' + doc + b',"x":01}', b'{"vc_document":' + doc + b',"x":"\\q"}', b'{"x":"\\ud800"}', b'{"x":1.5e+3}']
    return out


def main():
    reg = H.registry()
    cases = []
    for i, b in enumerate(bodies()):
        st, body = O.answer(b, reg)
        cases.append({"name": "req_%02d" % i, "body_hex": b.hex(), "expect_status": 200 if st == O.OK else 400,
                      "expect_body": body.decode("utf-8")})
    out = {"registry": [{"did": d, "pk": reg[d].hex()} for d in sorted(reg)], "cases": cases}
    with open(os.path.join(HERE, "verify_request_cases.json"), "w") as f:
        json.dump(out, f, indent=1, ensure_ascii=False)
        f.write("\n")


if __name__ == "__main__":
    main()
