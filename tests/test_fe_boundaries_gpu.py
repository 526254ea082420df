"""The field and scalar routines as the sm_90a kernels inline them — the inline-PTX carry chains of afc_fe.cuh, and the
AFC_FOLD_SHIFT and AFC_FE_KARATSUBA alternatives — through the tests/devsim harness, against Python integers bit for bit:
the boundary operands of tests/fe_cases.py, then 10^7 device-generated random items per operation checked against the
portable twins in the same kernel, with every 1000th item's output checked against Python integers."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import fe_cases as FC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEVSIM = os.path.join(ROOT, "tests", "devsim")
BUILDS = {"default": "libafc_devsim.so", "foldshift": "libafc_devsim_foldshift.so", "karatsuba": "libafc_devsim_kara.so"}
ALL_OPS = list(range(FC.OP_COUNT))
BULK_N, BULK_STRIDE = 10_000_000, 1000
SLOW = (FC.OP_INVERT, FC.OP_POW22523)       # exponentiation chains: checked as residues on random inputs


@pytest.fixture(scope="module")
def libs():
    subprocess.check_call(["make", "-s", "-C", DEVSIM])
    out = {}
    for name, so in BUILDS.items():
        lib = C.CDLL(os.path.join(DEVSIM, so))
        lib.devsim_run.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64]
        lib.devsim_bulk.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]
        assert lib.devsim_op_count() == FC.OP_COUNT
        out[name] = lib
    return out


@pytest.fixture(scope="module")
def cases():
    c = FC.all_cases()
    # expected words once, shared by the three builds
    return {op: (items, FC.pack(op, items), [FC.expected(op, x) for x in items]) for op, items in c.items()}


@pytest.fixture(scope="module")
def bulk_expect():
    """Per operation: the regenerated items devsim_bulk keeps, and their integer results."""
    out = {}
    idx = range(0, BULK_N, BULK_STRIDE)
    for op in ALL_OPS:
        items = FC.device_items(op, 0xB0 + op, idx)
        out[op] = (items, None if op in SLOW else [FC.expected(op, x) for x in items])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("build", list(BUILDS))
def test_constructed_cases(libs, cases, build):
    lib = libs[build]
    errs = []
    for op in ALL_OPS:
        items, words, exp = cases[op]
        out = np.zeros((len(items), 16), dtype=np.uint32)
        assert lib.devsim_run(op, words.ctypes.data, out.ctypes.data, len(items)) == 0, FC.OP_NAMES[op]
        got = FC.unpack_out(out)
        bad = [(x, g) for x, g, e in zip(items, got, exp) if g != e]
        if bad:
            errs.append(FC.describe(op, bad, len(items)))
    assert not errs, "%s build:\n%s" % (build, "\n".join(errs))


@pytest.mark.gpu
@pytest.mark.parametrize("build", list(BUILDS))
def test_bulk_random(libs, bulk_expect, build):
    lib = libs[build]
    errs = []
    for op in ALL_OPS:
        items, exp = bulk_expect[op]
        samples = np.zeros((len(items), 16), dtype=np.uint32)
        stats = np.zeros(2, dtype=np.uint64)
        assert lib.devsim_bulk(op, 0xB0 + op, BULK_N, BULK_STRIDE, samples.ctypes.data, stats.ctypes.data) == 0
        if stats[0]:
            errs.append("%s: %d of %d items differ from the portable twin, first at index %d"
                        % (FC.OP_NAMES[op], int(stats[0]), BULK_N, int(stats[1])))
        got = FC.unpack_out(samples)
        if exp is None:
            bad = FC.mismatches(op, items, got, exact=False)
        else:
            bad = [(x, g) for x, g, e in zip(items, got, exp) if g != e]
        if bad:
            errs.append(FC.describe(op, bad, len(items)))
    assert not errs, "%s build:\n%s" % (build, "\n".join(errs))


@pytest.mark.gpu
def test_unknown_operation_is_refused(libs):
    out = np.zeros((1, 16), dtype=np.uint32)
    inp = np.zeros((1, 32), dtype=np.uint32)
    for lib in libs.values():
        for op in (-1, FC.OP_COUNT):
            assert lib.devsim_run(op, inp.ctypes.data, out.ctypes.data, 1) != 0
