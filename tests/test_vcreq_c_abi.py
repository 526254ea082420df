"""afc_vc_verify_request_batch through a plain-C caller (tests/c_abi/verify_request.c): compiled as C99 with -pedantic against
include/afcrypto.h alone — what a cgo binding amounts to — into a temporary directory, then run on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _compile(out):
    lib = os.path.join(ROOT, "agentfield_b200")
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", out,
                           os.path.join(ROOT, "tests", "c_abi", "verify_request.c"), "-L" + lib, "-lafcrypto", "-Wl,-rpath," + lib])


def test_verify_request_caller_compiles_against_the_header(tmp_path):
    _compile(str(tmp_path / "verify_request"))


@pytest.mark.gpu
def test_verify_request_caller_passes(tmp_path):
    exe = str(tmp_path / "verify_request")
    _compile(exe)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "verify_request ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
