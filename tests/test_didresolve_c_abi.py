"""afc_did_directory_set_identities and afc_did_resolve_batch through a plain-C caller (tests/c_abi/did_resolve.c): compiled as C99 with -pedantic
against include/afcrypto.h alone — what a cgo binding amounts to — into a temporary directory, then run on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _compile(out):
    lib = os.path.join(ROOT, "agentfield_b200")
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", out,
                           os.path.join(ROOT, "tests", "c_abi", "did_resolve.c"), "-L" + lib, "-lafcrypto", "-Wl,-rpath," + lib])


def test_did_resolve_caller_compiles_against_the_header(tmp_path):
    _compile(str(tmp_path / "did_resolve"))


@pytest.mark.gpu
def test_did_resolve_caller_passes(tmp_path):
    exe = str(tmp_path / "did_resolve")
    _compile(exe)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "did_resolve ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
