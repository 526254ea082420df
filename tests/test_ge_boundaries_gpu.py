"""The group routines of afc_ge.cuh and the scalar recodings of afc_sc.cuh as the sm_90a kernels inline them — over the PTX
field paths of the default build and of the AFC_FOLD_SHIFT and AFC_FE_KARATSUBA builds — through the tests/devsim harness:
  * every constructed case of tests/ge_cases.py, bit for bit against the CPU build of the same harness (the portable
    twins), whose outputs are checked by value against big-integer Edwards arithmetic;
  * then 10^6 device-generated items per operation (10^5 for the key-table rows and ge_small_multiple), each run through
    the product form and the portable twin in the same kernel with zero differences allowed, and every 1000th output
    checked the same way: bit for bit against the CPU build, whose output is checked by value."""
import ctypes as C
import os

import numpy as np
import pytest

import ge_cases as GC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEVSIM = os.path.join(ROOT, "tests", "devsim")
BUILDS = {"default": "libafc_ge.so", "foldshift": "libafc_ge_foldshift.so", "karatsuba": "libafc_ge_kara.so"}
ALL_OPS = list(range(GC.GE_OP_COUNT))
BULK_STRIDE = 1000
BULK_N = {op: 100_000 if op in (GC.GE_KEY_ROWS, GC.GE_SMALL_MULT, GC.GE_SMALL_MULT_CALL) else 1_000_000 for op in ALL_OPS}


def bulk_seed(op):
    return 0xD0 + op


@pytest.fixture(scope="module")
def libs():
    # build() compiles these (tests/devsim/ge.mk); the test only loads them, so it writes nothing into the tree
    out = {}
    for name, so in BUILDS.items():
        path = os.path.join(DEVSIM, so)
        assert os.path.exists(path), "%s is missing: build() makes it (make -C tests/devsim -f ge.mk)" % path
        lib = C.CDLL(path)
        lib.ge_run.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64]
        lib.ge_bulk.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]
        GC.check_widths(lib)
        out[name] = lib
    return out


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return GC.build_host_lib(str(tmp_path_factory.mktemp("gesim")))


@pytest.fixture(scope="module")
def cases(host):
    """Per operation: input words, the portable outputs and the errors Python finds in them (none expected)."""
    out = {}
    for op, items in GC.all_cases().items():
        x = GC.pack(op, items)
        y = GC.run(host, op, x)
        out[op] = (x, y, GC.mismatches(op, x, y, [e for _, e in items]))
    return out


@pytest.fixture(scope="module")
def bulk_expect(host):
    """Per operation: the regenerated items ge_bulk keeps, their portable outputs and the errors Python finds in them."""
    out = {}
    for op in ALL_OPS:
        x = GC.device_items(op, bulk_seed(op), range(0, BULK_N[op], BULK_STRIDE))
        y = GC.run(host, op, x)
        out[op] = (x, y, GC.mismatches(op, x, y))
    return out


def _device_vs_portable(op, x, got, want, label):
    diff = np.nonzero((got != want).any(axis=1))[0]
    if not len(diff):
        return None
    bad = GC.mismatches(op, x[diff], got[diff])
    i = int(diff[0])
    return "%s: %d of %d %s differ from the portable build (first item %d; %d also wrong by value%s)" % (
        GC.OP_NAMES[op], len(diff), len(x), label, i, len(bad), (": " + bad[0][1]) if bad else "")


@pytest.mark.gpu
@pytest.mark.parametrize("build", list(BUILDS))
def test_constructed_cases(libs, cases, build):
    lib = libs[build]
    errs = []
    for op in ALL_OPS:
        x, want, bad_portable = cases[op]
        assert not bad_portable, GC.describe(op, bad_portable, len(x), x)
        got = np.zeros_like(want)
        assert lib.ge_run(op, x.ctypes.data, got.ctypes.data, len(x)) == 0, GC.OP_NAMES[op]
        err = _device_vs_portable(op, x, got, want, "constructed cases")
        if err:
            errs.append(err)
    assert not errs, "%s build:\n%s" % (build, "\n".join(errs))


@pytest.mark.gpu
@pytest.mark.parametrize("build", list(BUILDS))
def test_bulk_random(libs, bulk_expect, build):
    lib = libs[build]
    errs = []
    for op in ALL_OPS:
        x, want, bad_portable = bulk_expect[op]
        assert not bad_portable, GC.describe(op, bad_portable, len(x), x)
        got = np.zeros_like(want)
        stats = np.zeros(2, dtype=np.uint64)
        assert lib.ge_bulk(op, bulk_seed(op), BULK_N[op], BULK_STRIDE, got.ctypes.data, stats.ctypes.data) == 0
        if stats[0]:
            errs.append("%s: %d of %d items differ from the portable twin, first at index %d"
                        % (GC.OP_NAMES[op], int(stats[0]), BULK_N[op], int(stats[1])))
        err = _device_vs_portable(op, x, got, want, "kept outputs")
        if err:
            errs.append(err)
    assert not errs, "%s build:\n%s" % (build, "\n".join(errs))


@pytest.mark.gpu
def test_items_outside_the_domain_are_refused(libs):
    for lib in libs.values():
        for op in (-1, GC.GE_OP_COUNT):
            out = np.zeros((1, 8), dtype=np.uint32)
            assert lib.ge_run(op, np.zeros((1, 32), dtype=np.uint32).ctypes.data, out.ctypes.data, 1) != 0
        x = np.zeros((1, GC.IN_WORDS[GC.GE_GROUP_KC]), dtype=np.uint32)     # G = 0
        y = np.zeros((1, GC.OUT_WORDS[GC.GE_GROUP_KC]), dtype=np.uint32)
        assert lib.ge_run(GC.GE_GROUP_KC, x.ctypes.data, y.ctypes.data, 1) != 0
