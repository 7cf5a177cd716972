"""CPU-only: the asynchronous packed decode, Wrap and Unwrap calls (lz4b200_decode_batch_packed_to_device_async,
lz4b200_wrap_batch_packed_from_device_async, lz4b200_unwrap_batch_to_device_async,
lz4b200_unwrap_batch_packed_to_device_async) are declared, bound and exported with the parameter lists of their
synchronous forms; without a device they fail and write nothing; the Python wrappers refuse host tensors that are not
page-locked before the library sees them; the C++ mirror's methods compile against the header."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# each asynchronous call and the synchronous form whose parameter list it takes
PAIRS = {
    "lz4b200_decode_batch_packed_to_device_async": "lz4b200_decode_batch_packed_to_device",
    "lz4b200_wrap_batch_packed_from_device_async": "lz4b200_wrap_batch_packed_from_device",
    "lz4b200_unwrap_batch_to_device_async": "lz4b200_unwrap_batch_to_device",
    "lz4b200_unwrap_batch_packed_to_device_async": "lz4b200_unwrap_batch_packed_to_device",
}


@pytest.fixture(scope="module")
def lib():
    from lz4net_b200 import build, native
    build.build()
    return native.lib()


def test_symbols_are_declared_bound_and_exported_like_the_synchronous_calls(lib):
    from lz4net_b200 import native
    hdr = open(os.path.join(ROOT, "include", "lz4b200.h")).read()
    for name, sync in PAIRS.items():
        assert re.search(r"\bint\s+%s\s*\(" % name, hdr), name
        assert hasattr(lib, name), name
        assert native.SIGNATURES[name] == native.SIGNATURES[sync], name
    # the CUDA-graph paragraph names every asynchronous call among those that refuse a capturing stream
    graphs = hdr[hdr.index("---- CUDA graphs"):hdr.index("int lz4b200_reserve(")]
    for name in PAIRS:
        assert name[len("lz4b200_"):] in re.sub(r"\s+", " ", graphs), name


def test_without_a_device_every_call_fails_and_writes_nothing(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lz4net_b200 import native
    h = C.c_void_p()
    assert lib.lz4b200_create(C.byref(h), 0) == native.E_NODEVICE and not h.value
    src = np.frombuffer(b"\x02\0\0\0\x02\0\0\0ab" + bytes(16), np.uint8).copy()
    so, sl, cap = np.zeros(1, np.int64), np.array([10], np.int32), np.array([64], np.int32)
    dst = np.full(64, 0xEE, np.uint8)
    off, out = np.full(2, -7, np.int64), np.full(1, 12345, np.int32)
    p = lambda a: a.ctypes.data                                                                 # noqa: E731
    calls = {
        "lz4b200_decode_batch_packed_to_device_async": (h, p(src), p(so), p(sl), p(dst), 64, p(off), p(out), 1, None),
        "lz4b200_wrap_batch_packed_from_device_async": (h, p(src), p(so), p(sl), 0, p(dst), 64, p(off), p(out), 1, None),
        "lz4b200_unwrap_batch_to_device_async": (h, p(src), p(so), p(sl), p(dst), p(so), p(cap), p(out), 1, None),
        "lz4b200_unwrap_batch_packed_to_device_async": (h, p(src), p(so), p(sl), p(dst), 64, p(off), p(out), 1, None),
    }
    for name, args in calls.items():
        assert getattr(lib, name)(*args) < 0 and native.last_error(), name
        assert (dst == 0xEE).all() and (off == -7).all() and out[0] == 12345, name


class _NoContext:
    handle = None


def test_python_wrappers_refuse_host_tensors_that_are_not_page_locked(lib):
    """Each refusal is a TypeError raised before the library is called (the context here is no context at all)."""
    import torch
    from lz4net_b200 import batch
    n = 2
    so, sl, cap = np.zeros(n, np.int64), np.full(n, 9, np.int32), np.full(n, 32, np.int32)
    pageable = torch.zeros(64, dtype=torch.uint8)
    off, out = torch.zeros(n + 1, dtype=torch.int64), torch.zeros(n, dtype=torch.int32)
    raw = torch.zeros(64, dtype=torch.uint8)
    nc = _NoContext()
    with pytest.raises(TypeError, match="dst: expected a page-locked CPU tensor"):
        batch.wrap_to_host_packed_async(nc, raw, so, sl, pageable, off, out)
    with pytest.raises(TypeError, match="packets: expected a page-locked CPU tensor"):
        batch.unwrap_to_device_async(nc, pageable, so, sl, raw, so, cap, out)
    with pytest.raises(TypeError, match="packets: expected a page-locked CPU tensor"):
        batch.unwrap_to_device_packed_async(nc, pageable, so, sl, raw, off, out)
    with pytest.raises(TypeError, match="comp: expected a page-locked CPU tensor"):
        batch.decode_from_host_packed_async(nc, pageable, so, sl, raw, off, out)
    with pytest.raises(TypeError):
        batch.unwrap_to_device_packed_async(nc, np.zeros(64, np.uint8), so, sl, raw, off, out)   # packets: numpy, not a tensor
    with pytest.raises(TypeError, match="dst: expected a contiguous"):
        batch.wrap_to_host_packed_async(nc, raw, so, sl, pageable.to(torch.int8), off, out)      # dst: not uint8


def test_cpp_mirror_methods_compile_against_the_header(tmp_path):
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c",
                           os.path.join(ROOT, "tests", "cpp", "async_wrap_mirror.cpp"), "-o", str(tmp_path / "async_wrap_mirror.o")])
