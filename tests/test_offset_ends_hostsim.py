"""offset_ends (agentfield_b200/csrc/afc_common.cuh), compiled for the CPU (tests/hostsim/hostsim_offset_ends.cpp), against a plain restatement:
for the span list of every call that sizes its output from the ends of its offset arrays, on seeded random arrays, for batches that start
past item 0 and past record 0, and for backwards index ranges, where the indirect array is not read at all (it is passed as NULL)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (stride, via) of each span, as afcrypto.cu lists them per call
SPANS = {
    "stored, JSON, audit": [(1, -1)],
    "issue": [(14, -1)],
    "webhook": [(8, -1), (1, -1)],
    "workflow": [(7, -1), (1, -1), (2, 1)],
    "chain": [(7, -1), (1, -1), (2, 1), (2, -1), (13, 1)],
    "register": [(1, -1), (2, -1), (1, 1)],
    "reregister": [(3, -1), (2, -1), (1, 1), (2, -1), (5, 3)],
    "resolve": [(1, -1)],
}


@pytest.fixture(scope="module")
def oe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("oesim") / "libafc_oesim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_offset_ends.cpp")])
    return C.CDLL(out)


def _ref(spans, arrays, n):
    out = []
    for (stride, via), a in zip(spans, arrays):
        lo, hi = (0, n) if via < 0 else (out[2 * via], out[2 * via + 1])
        out += [0, 0] if hi < lo else [int(a[stride * lo]), int(a[stride * hi])]
    return out


def _run(oe, spans, arrays, n):
    k = len(spans)
    offs = (C.c_void_p * k)(*[None if a is None else a.ctypes.data for a in arrays])
    strides = (C.c_uint32 * k)(*[s for s, _ in spans])
    vias = (C.c_int32 * k)(*[v for _, v in spans])
    out = (C.c_uint64 * (2 * k))()
    oe.hs_offset_ends(offs, strides, vias, k, C.c_uint32(n), out)
    return list(out)


def _arrays(rng, spans, n, backwards):
    """One batch of n items starting at item i0 of a larger one: a direct array is sliced at its stride times i0, an indirect one is
    indexed by the absolute indices its via span reads and is passed whole.  backwards: each via array's last end drops below its first
    (the indirect arrays are then NULL)."""
    i0 = int(rng.integers(0, 5))
    arrays, lengths = [], {}
    for j, (stride, via) in enumerate(spans):
        if via < 0:
            index = any(v == j for _, v in spans)          # its words index another array: small, and never below 1
            base = int(rng.integers(1, 50)) if index else int(rng.integers(0, 1 << 40))
            steps = rng.integers(0, 4 if index else 1000, stride * (i0 + n))
            a = np.concatenate([[base], steps]).cumsum().astype(np.uint64)
            a = np.ascontiguousarray(a[stride * i0:])
            if backwards and index:
                a[stride * n] = int(rng.integers(0, int(a[0])))
            elif index and rng.random() < 0.2:
                a[stride * n] = a[0]                        # an empty index range still reads both words
            arrays.append(a)
            lengths[j] = int(a.max())
        else:
            if backwards:
                arrays.append(None)
            else:
                m = stride * lengths[via] + 1
                arrays.append(np.sort(rng.integers(0, 1 << 50, m, dtype=np.uint64)))
    return arrays


@pytest.mark.parametrize("call", sorted(SPANS))
def test_offset_ends_equals_restatement(oe, call):
    spans = SPANS[call]
    rng = np.random.default_rng(0x0E5 + len(call))
    has_via = any(v >= 0 for _, v in spans)
    for trial in range(300):
        n = int(rng.integers(1, 40))
        backwards = has_via and trial % 3 == 2
        arrays = _arrays(rng, spans, n, backwards)
        got = _run(oe, spans, arrays, n)
        assert got == _ref(spans, arrays, n), (call, trial)
        if backwards:
            for j, (_, via) in enumerate(spans):
                if via >= 0:
                    assert got[2 * via + 1] < got[2 * via] and got[2 * j:2 * j + 2] == [0, 0], (call, trial)
