"""The group routines of afc_ge.cuh and the scalar recodings of afc_sc.cuh, compiled for the CPU through the tests/devsim
harness (the portable twins), against big-integer Edwards arithmetic at the points random keys never reach: the torsion
points and x = 0 in every encoding, decodings that need the sqrt(-1) correction, sums and differences of every pair of
exceptional points at weakly reduced projective scales, groups of encodings at every size the kernels use, key-table rows
of small-order and mixed-order keys, and recodings whose carries run into the top digit.  The same cases run on the
device in tests/test_ge_boundaries_gpu.py."""
import os
import re

import numpy as np
import pytest

import ge_cases as GC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL_OPS = list(range(GC.GE_OP_COUNT))
# random items per operation: 10^4, fewer where one item is many group operations to replay in Python (groups of encodings,
# runs of table entries, key-table rows, double-and-add chains), to keep this file within about 25 s
N_RANDOM = {GC.GE_GROUP_KC: 1500, GC.GE_GROUP_SIGN: 6000, GC.GE_GROUP_SIGN2: 3000, GC.GE_AFFINE_RUN: 400,
            GC.GE_AFFINE_RUN_CALL: 400, GC.GE_AFFINE_FWDBWD: 800, GC.GE_KEY_ROWS: 200, GC.GE_SMALL_MULT: 3000,
            GC.GE_SMALL_MULT_CALL: 3000}


@pytest.fixture(scope="module")
def gs(tmp_path_factory):
    return GC.build_host_lib(str(tmp_path_factory.mktemp("gesim")))


@pytest.fixture(scope="module")
def cases():
    return GC.all_cases()


def test_harness_mirrors_the_kernels():
    # ge_ops.cuh runs each routine at the group sizes, slice shape and field policies k_ed25519.cu gives it
    src = open(os.path.join(ROOT, "agentfield_b200", "csrc", "k_ed25519.cu")).read()
    assert re.search(r"#define AFC_KC_GMAX %d\b" % GC.KC_GMAX, src)
    assert re.search(r"constexpr int SIGN_GMAX = %d;" % GC.SIGN_GMAX, src)
    assert re.search(r"#define AFC_KEYROW_PARTS %d\b" % GC.KR_PARTS, src)
    assert re.search(r"#define AFC_SIGN_FE FeCall\b", src)
    assert re.search(r"#define AFC_BASES_FE FeInline\b", src) and re.search(r"#define AFC_ROWS_FE FeInline\b", src)
    assert "ge_encode_group<FeInline, KC_GMAX>" in src and "ge_encode_group<AFC_SIGN_FE, 2 * SIGN_GMAX>" in src
    assert "ge_encode_group<AFC_SIGN_FE, SIGN_GMAX>" in src
    assert "ge_key_slice_start<FeCall, KR_PARTS>" in src and "ge_build_base_chunk<FeCall>" in src
    ge = open(os.path.join(ROOT, "agentfield_b200", "csrc", "afc_ge.cuh")).read()
    assert re.search(r"BASE_CHUNK = 64;", ge) and re.search(r"#define AFC_KEYROW_CHUNK 64\b", ge)


def test_constructed_cases_reach_their_branches(cases):
    br = GC.Branches()
    for row, _ in cases[GC.GE_DECODE]:
        want = GC.decode(GC.get(row, 0))
        assert GC.decode_replay(GC.get(row, 0), br) == want      # the replay is the oracle's decoding
    missed = {b: why for b, why in GC.DECODE_BRANCHES.items() if br[b] == 0}
    assert not missed, missed
    assert br["decode.reject"] >= 64 and br["decode.sqrtm1"] >= 64, dict(br)
    # the other edges the cases name
    ds = [GC.s32(r[192]) for r, _ in cases[GC.GE_CT_SELECT]]
    assert ds.count(8) >= 2 and ds.count(-8) >= 2 and ds.count(0) >= 2
    assert sum(int(r[32]) >> 21 for r, _ in cases[GC.GE_SMALL_MULT]) >= 10
    for op, gmax in GC.GMAX.items():
        assert {int(r[0]) for r, _ in cases[op]} == set(range(1, gmax + 1))
        assert any(1 in e[1:] for _, e in cases[op])                     # padding members after real ones
    keys = {GC.get(r, 0) for r, _ in cases[GC.GE_KEY_ROWS]}
    assert sum(GC.decode(k) is None for k in keys) == 1 and len(keys) >= 20
    tops = [GC.get(r, 0) for r, _ in cases[GC.GE_RECODE] if int(r[8]) >= 16]
    assert 2**253 - 1 in tops


def test_recoding_geometry_from_integers():
    # base_table_top_max(w) bounds the top digit of every s < 2^253 and base_table_entries(w) holds that digit
    for w in range(16, 23):
        _, rows, c, _ = GC.recode_geometry(w)
        tm = GC.top_max(w)
        assert (2**253 - 1 + c) >> (w * (rows - 1)) == tm and (2**252 + c) >> (w * (rows - 1)) <= tm
        assert GC.table_entries(w) - (rows - 1) * (1 << (w - 1)) >= tm
        assert tm <= 1 << (w - 1)


@pytest.mark.parametrize("op", ALL_OPS, ids=GC.OP_NAMES)
def test_constructed_cases(gs, cases, op):
    items = cases[op]
    assert items
    x = GC.pack(op, items)
    y = GC.run(gs, op, x)
    bad = GC.mismatches(op, x, y, [e for _, e in items])
    assert not bad, GC.describe(op, bad, len(items), x)


@pytest.mark.parametrize("op", ALL_OPS, ids=GC.OP_NAMES)
def test_random(gs, op):
    n = N_RANDOM.get(op, 10_000)
    x = GC.device_items(op, 0xC0 + op, range(n))
    y = GC.run(gs, op, x)
    bad = GC.mismatches(op, x, y)
    assert not bad, GC.describe(op, bad, n, x)


def test_items_outside_the_domain_are_refused(gs):
    for op, word, val in ((GC.GE_GROUP_KC, 0, 0), (GC.GE_GROUP_SIGN, 0, 9), (GC.GE_KEY_ROWS, 8, 32), (GC.GE_KEY_ROWS, 9, 3),
                          (GC.GE_RECODE, 8, 3), (GC.GE_RECODE, 8, 23)):
        x = np.zeros((1, GC.IN_WORDS[op]), dtype=np.uint32)
        if op == GC.GE_KEY_ROWS:
            x[0, 9] = 1                              # one stage, row 0: in the domain but for the word under test
        x[0, word] = val
        y = np.zeros((1, GC.OUT_WORDS[op]), dtype=np.uint32)
        assert gs.ge_run(op, x.ctypes.data, y.ctypes.data, 1) == 1, (GC.OP_NAMES[op], word, val)
    y = np.zeros((1, 8), dtype=np.uint32)
    assert gs.ge_run(GC.GE_OP_COUNT, np.zeros((1, 32), dtype=np.uint32).ctypes.data, y.ctypes.data, 1) == 1


def test_device_generator_replica():
    # ge_bulk's kept items are regenerated in Python; the replica must draw what the device draws, in the domain
    x = GC.device_items(GC.GE_ADDSUB, 7, range(3000))
    limbs = x[:, :64].ravel()
    zeros, ones = (limbs == 0).mean(), (limbs == 0xFFFFFFFF).mean()
    assert 0.05 < zeros < 0.075 and 0.11 < ones < 0.14, (zeros, ones)
    assert set(x[:, 64]) == {0, 1}
    r = GC.device_items(GC.GE_RECODE, 7, range(3000))
    assert set(r[:, 8]) == set(GC.RECODE_KINDS)
    c = GC.device_items(GC.GE_CT_SELECT, 7, range(3000))
    assert {GC.s32(v) for v in c[:, 192]} == set(range(-8, 9))
