"""The recoding of the table-driven verify's radix-2^w fixed-base table (afc_sc.cuh, compiled for the CPU from
tests/hostsim/hostsim_wide.cpp) replayed against Python integers at every window the library accepts, and the table geometry that
bounds its gathers."""
import ctypes as C
import os
import subprocess

import pytest

from oracle import go_ed25519 as G
from wide_base_cases import WINDOWS, compose, recode, rows, scalars

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def widesim(tmp_path_factory):
    """TEST-ONLY CPU build of the recoding (tests/hostsim/hostsim_wide.cpp), compiled into a temporary directory."""
    out = str(tmp_path_factory.mktemp("widesim") / "libafc_widesim.so")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas", "-o", out,
                           os.path.join(ROOT, "tests", "hostsim", "hostsim_wide.cpp")])
    return C.CDLL(out)


def _digits(lib, w, s):
    out = (C.c_int32 * 32)()
    top, entries = C.c_int(), C.c_uint64()
    r = lib.hs_wide_digits(w, s.to_bytes(32, "little"), out, C.byref(top), C.byref(entries))
    return list(out[:r]), top.value, entries.value


def test_wide_recoding_matches_integers(widesim):
    for w in WINDOWS:
        h = 1 << (w - 1)
        cases = scalars(w)
        assert len(cases) >= rows(w) + 6, w
        top_max = recode(2**253 - 1, w)[-1]
        for name, s in cases.items():
            d, top, entries = _digits(widesim, w, s)
            assert d == recode(s, w), (w, name)
            assert compose(d, w) == s, (w, name)
            assert all(-h <= x < h for x in d[:-1]) and 0 <= d[-1] <= top_max <= h, (w, name)
            assert top == top_max and entries == (rows(w) - 1) * h + -(-top_max // 64) * 64, w
        # the named corners are reached
        assert set(recode(cases["every digit -2^(w-1)"], w)[:-1]) == {-h}
        assert set(recode(cases["every digit 2^(w-1)-1"], w)[:-1]) == {h - 1}
        assert recode(cases["carries into the top row"], w)[-1] == 1
        assert recode(G.L - 1, w)[-1] <= top_max


def test_wide_recoding_at_16_is_the_radix_65536_recoding(widesim):
    """w = 16 reads the radix-65536 table the library builds at init (and falls back to): same digits as sc_recode65536."""
    for s in list(scalars(16).values()) + [G.L - 1]:
        t = s + int("8000" * 16, 16)
        old = [((t >> (16 * i)) & 0xffff) - 0x8000 for i in range(16)]
        d, _, _ = _digits(widesim, 16, s)
        assert compose(old, 16) == s and d[:-1] == old[:-1] and d[-1] == old[-1], hex(s)
