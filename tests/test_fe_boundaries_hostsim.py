"""The field and scalar routines (agentfield_b200/csrc/afc_fe.cuh, afc_sc.cuh), compiled for the CPU through the tests/devsim
harness (the portable twins), against Python integers at the carries and reductions random operands never reach: the
second wrap of fe_add / fe_fold16 / fe_mul, the second borrow of fe_sub / fe_addsub_m, fe_towords either side of p, 2p and
2^256, Barrett's correction.  The same cases run on the device in tests/test_fe_boundaries_gpu.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import fe_cases as FC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_OPS = [op for op in range(FC.OP_COUNT) if op not in FC.DEVICE_ONLY]


@pytest.fixture(scope="module")
def ds(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("devsim") / "libafc_devsim_host.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "devsim", "devsim_host.cpp")])
    lib = C.CDLL(out)
    lib.devsim_run.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64]
    assert lib.devsim_op_count() == FC.OP_COUNT
    return lib


def run(lib, op, words):
    words = np.ascontiguousarray(words, dtype=np.uint32)
    out = np.zeros((len(words), 16), dtype=np.uint32)
    assert lib.devsim_run(op, words.ctypes.data, out.ctypes.data, len(words)) == 0, FC.OP_NAMES[op]
    return FC.unpack_out(out)


@pytest.fixture(scope="module")
def cases():
    return FC.all_cases()


def test_constructed_cases_reach_their_branches(cases):
    br = FC.Branches()
    for op, items in cases.items():
        for x in items:
            FC.count_branches(op, x, br)
    missed = {b: why for b, why in FC.REQUIRED_BRANCHES.items() if br[b] == 0}
    assert not missed, missed
    assert br["sc.corr0"] > 0 and br["fold.wrap2"] >= 38 and br["add.wrap2"] >= 37 and br["sub.borrow2"] >= 37, dict(br)
    assert len(cases[FC.OP_MUL]) >= 2**16 + 96


def test_barrett_estimate_is_never_two_low():
    # So the second conditional subtraction in sc_reduce512 cannot fire for any 512-bit input, and no case can reach it.
    assert FC.barrett_max_deficit() < 1
    assert float(FC.barrett_max_deficit()) < 0.23


def test_replays_are_the_integer_results():
    # the bit-exact expectations are replays of the limb algorithms; each must also be the right residue
    rng = np.random.default_rng(3)
    for x, y in zip(*(rng.integers(0, 2**63, (2, 500, 5)).tolist())):
        a = sum(v << (52 * i) for i, v in enumerate(x)) & FC.M256
        b = sum(v << (52 * i) for i, v in enumerate(y)) & FC.M256
        assert FC.add_ref(a, b) % FC.P == (a + b) % FC.P and FC.sub_ref(a, b) % FC.P == (a - b) % FC.P
        assert FC.mul_ref(a, b) % FC.P == a * b % FC.P and FC.fold_ref(a << 256 | b) % FC.P == (a << 256 | b) % FC.P
        assert FC.barrett_ref(a * b) == a * b % FC.L


@pytest.mark.parametrize("op", HOST_OPS, ids=[FC.OP_NAMES[o] for o in HOST_OPS])
def test_constructed_cases(ds, cases, op):
    items = cases[op]
    assert items
    got = run(ds, op, FC.pack(op, items))
    bad = FC.mismatches(op, items, got)
    assert not bad, FC.describe(op, bad, len(items))


@pytest.mark.parametrize("op", HOST_OPS, ids=[FC.OP_NAMES[o] for o in HOST_OPS])
def test_random(ds, op):
    exact = op not in (FC.OP_INVERT, FC.OP_POW22523)
    n = 100_000 if exact else 10_000
    words, items = FC.random_items(op, n, seed=1000 + op)
    got = run(ds, op, words)
    bad = FC.mismatches(op, items, got, exact)
    assert not bad, FC.describe(op, bad, n)


def test_device_only_operations_are_refused(ds):
    for op in sorted(FC.DEVICE_ONLY) + [FC.OP_COUNT, -1]:
        out = np.zeros((1, 16), dtype=np.uint32)
        assert ds.devsim_run(op, np.zeros((1, 32), dtype=np.uint32).ctypes.data, out.ctypes.data, 1) == 1


def test_device_generator_replica():
    # devsim_bulk's kept items are regenerated in Python; the replica's distribution must be what the device draws
    items = FC.device_items(FC.OP_MUL_WIDE, 7, range(2000))
    limbs = [(v >> (32 * k)) & 0xFFFFFFFF for x in items for v in x for k in range(8)]
    zeros, ones = limbs.count(0) / len(limbs), limbs.count(0xFFFFFFFF) / len(limbs)
    assert 0.05 < zeros < 0.075 and 0.11 < ones < 0.14, (zeros, ones)
