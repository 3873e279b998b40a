"""The engine's owners of device memory, events and streams (tardis_b200/csrc/device_buffer.cuh), on the CPU.

tests/device_buffer_shim.cpp compiles the header with g++ against counting stand-ins for the CUDA runtime calls it makes
and logs every call: "M3" is cudaMalloc handing out id 3 and "F3" its cudaFree, E / e and S / s the same for events and
streams, "X" a free or destroy of something that is not live (a double free, or a null handle)."""
import collections
import ctypes as C
import os
import subprocess

import pytest

from tardis_b200._build import find_nvcc

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TB200_ERR_CUDA = 100  # include/tardis_b200.h


@pytest.fixture(scope="module")
def shim():
    out = os.path.join(HERE, "_shim", "libdevice_buffer_shim.so")
    src = os.path.join(HERE, "device_buffer_shim.cpp")
    deps = [src, __file__, os.path.join(ROOT, "tardis_b200", "csrc", "device_buffer.cuh"), os.path.join(ROOT, "include", "tardis_b200.h")]
    cuda_include = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(find_nvcc()))), "include")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(d) for d in deps):
        # -Bsymbolic: the header's calls go to the stand-ins even when the process has loaded the real cudart globally
        # (importing torch does)
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wl,-Bsymbolic", "-I", cuda_include, "-o", out, src],
                       check=True)
    lib = C.CDLL(out)
    lib.shim_log.restype = C.c_char_p
    lib.shim_last_error.restype = C.c_char_p
    lib.shim_ensure_fails.argtypes = [C.POINTER(C.c_int), C.POINTER(C.c_longlong)]
    return lib


def run(shim, scenario, *args):
    """-> (what the scenario returned, its call log)"""
    shim.shim_reset()
    rc = getattr(shim, scenario)(*args)
    assert shim.shim_live() == 0, (scenario, shim.shim_log())
    return rc, shim.shim_log().decode()


def test_a_struct_of_owners_frees_each_once_buffers_first(shim):
    """Streams and events declared before the buffers (as in tb200_engine) go after them; owners that never got a
    handle make no call."""
    rc, log = run(shim, "shim_owners_struct")
    assert rc == 0
    assert log == "S1 E2 E3 M4 M5 M6 F6 F5 F4 e3 e2 s1"


def test_moves_transfer_ownership(shim):
    """Move construction, move assignment (which frees what the target held) and vector growth: every handle is
    released exactly once."""
    rc, log = run(shim, "shim_moves")
    assert rc == 0, f"check {rc} failed"
    calls = log.split()
    assert "X" not in calls
    made = [c[1:] for c in calls if c[0] in "MES"]
    gone = collections.Counter(c[1:] for c in calls if c[0] in "Fes")
    assert len(made) == 10 and gone == collections.Counter(made)
    assert calls.index("F2") < calls.index("M3")  # c = std::move(b) frees c's own buffer at once
    assert calls.index("e6") < calls.index("S7")  # g = std::move(f) destroys g's own event at once


def test_ensure_frees_before_it_grows_and_keeps_a_large_enough_buffer(shim):
    rc, log = run(shim, "shim_ensure_sizes")
    assert rc == 0, f"check {rc} failed"
    assert log == "M1 F1 M2 F2"


def test_failed_cudamalloc_leaves_the_buffer_empty(shim):
    p_null, n = C.c_int(0), C.c_longlong(-1)
    rc, log = run(shim, "shim_ensure_fails", C.byref(p_null), C.byref(n))
    assert rc == TB200_ERR_CUDA
    assert p_null.value == 1 and n.value == 0
    assert log == "M1 F1"
    assert shim.shim_last_error().decode() == "cudaMalloc: out of memory"
