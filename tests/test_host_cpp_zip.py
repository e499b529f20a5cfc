"""The C++ host mirror's byte, view, Boolean and FixedSizeBinary zip (arrow-rs_b200/host/test_host_zip.cpp): builds on CPU, refuses to run
without a GPU, and on a GPU the reference's tests re-expressed in C++ must pass."""
import ctypes as C
import os
import subprocess

import pytest

from acu import _abi as abi

HOST = os.path.join(abi.REPO, "arrow-rs_b200", "host")
BIN = os.path.join(HOST, "test_host_zip")


def test_host_zip_builds():
    subprocess.run(["make", "-s", "-C", HOST, "test_host_zip"], check=True)
    assert os.path.exists(BIN)


def test_host_zip_refuses_to_run_without_gpu():
    lib = abi.load_library()
    h = C.c_void_p()
    if lib.acu_ctx_create(0, C.byref(h)) == abi.OK:
        lib.acu_ctx_destroy(h)
        pytest.skip("CUDA device present")
    if not os.path.exists(BIN):
        subprocess.run(["make", "-s", "-C", HOST, "test_host_zip"], check=True)
    r = subprocess.run([BIN], capture_output=True, text=True)
    assert r.returncode == 77 and "no CPU fallback" in r.stdout


@pytest.mark.gpu
def test_host_zip_reference_tests_pass():
    if not os.path.exists(BIN):
        subprocess.run(["make", "-s", "-C", HOST, "test_host_zip"], check=True)
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
    assert "0 failed" in r.stdout
