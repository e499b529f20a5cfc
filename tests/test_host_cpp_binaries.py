"""The C++ host mirror's per-area test binaries (arrow-rs_b200/host/test_host_<area>.cpp), each the reference's tests of
that area re-expressed in C++: every one builds on CPU, refuses to run without a GPU, and passes on a GPU. test_host
itself is covered by test_host_cpp.py, which also writes its IPC fixture."""
import ctypes as C
import os
import subprocess

import pytest

from acu import _abi as abi

HOST = os.path.join(abi.REPO, "arrow-rs_b200", "host")
BINARIES = [
    "test_host_aggregate",  # min / max of string, string-view and boolean columns
    "test_host_bitwise",  # bitwise operations and product / bit aggregates
    "test_host_concat_elements",
    "test_host_decimal",
    "test_host_decimal_cast",
    "test_host_fixed_size_binary",  # FixedSizeBinary filter / take
    "test_host_like",  # the LIKE family
    "test_host_list",  # List / LargeList / FixedSizeList filter / take
    "test_host_run_end",  # RunEndEncoded filter / take
    "test_host_substring",  # length / substring
    "test_host_union",  # Struct and Union filter / take
    "test_host_zip",  # byte, view, Boolean and FixedSizeBinary zip
]


def _make(name):
    subprocess.run(["make", "-s", "-C", HOST, name], check=True)


@pytest.mark.parametrize("name", BINARIES)
def test_builds(name):
    _make(name)
    assert os.path.exists(os.path.join(HOST, name))


@pytest.mark.parametrize("name", BINARIES)
def test_refuses_to_run_without_gpu(name):
    lib = abi.load_library()
    h = C.c_void_p()
    if lib.acu_ctx_create(0, C.byref(h)) == abi.OK:
        lib.acu_ctx_destroy(h)
        pytest.skip("CUDA device present")
    if not os.path.exists(os.path.join(HOST, name)):
        _make(name)
    r = subprocess.run([os.path.join(HOST, name)], capture_output=True, text=True)
    assert r.returncode == 77 and "no CPU fallback" in r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("name", BINARIES)
def test_reference_tests_pass(name):
    if not os.path.exists(os.path.join(HOST, name)):
        _make(name)
    r = subprocess.run([os.path.join(HOST, name)], capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-1000:]
    assert "0 failed" in r.stdout
