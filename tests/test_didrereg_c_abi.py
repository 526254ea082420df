"""afc_did_reregister_batch through a plain-C caller (tests/c_abi/did_reregister.c): compiled as C99 with -pedantic against
include/afcrypto.h alone — what a cgo binding amounts to — into a temporary directory.  The bound checks run without a GPU (the caller
then exits 77); the rest runs on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _compile(out):
    lib = os.path.join(ROOT, "agentfield_b200")
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", out,
                           os.path.join(ROOT, "tests", "c_abi", "did_reregister.c"), "-L" + lib, "-lafcrypto", "-Wl,-rpath," + lib])


def test_did_reregister_bound_from_c(tmp_path):
    exe = str(tmp_path / "did_reregister")
    _compile(exe)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert "bound ok" in r.stdout and r.returncode in (0, 77), (r.returncode, r.stdout, r.stderr)


@pytest.mark.gpu
def test_did_reregister_caller_passes(tmp_path):
    exe = str(tmp_path / "did_reregister")
    _compile(exe)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "did_reregister ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
