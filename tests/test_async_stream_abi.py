"""CPU-only: the asynchronous LZ4Stream calls (lz4b200_stream_encode_from_device_async,
lz4b200_stream_decode_to_device_async) are declared, bound and exported; without a device they fail and write nothing;
the Python wrappers refuse host tensors that are not page-locked before the library sees them; the C++ mirror's methods
compile against the header."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("lz4b200_stream_encode_from_device_async", "lz4b200_stream_decode_to_device_async")


@pytest.fixture(scope="module")
def lib():
    from lz4net_b200 import build, native
    build.build()
    return native.lib()


def test_symbols_are_declared_bound_and_exported(lib):
    from lz4net_b200 import native
    hdr = open(os.path.join(ROOT, "include", "lz4b200.h")).read()
    P, I, L = C.c_void_p, C.c_int, C.c_int64
    want = {CALLS[0]: (I, [P, P, L, C.c_int32, I, P, L, P, P]), CALLS[1]: (I, [P, P, L, P, L, P, P])}
    for name in CALLS:
        assert re.search(r"\bint\s+%s\s*\(" % name, hdr), name
        assert hasattr(lib, name), name
        assert native.SIGNATURES[name] == want[name], name
    # the synchronous forms' leading parameters, then out_size and the stream
    assert native.SIGNATURES[CALLS[0]][1][:7] == native.SIGNATURES["lz4b200_stream_encode_from_device"][1][:7]
    assert native.SIGNATURES[CALLS[1]][1][:5] == native.SIGNATURES["lz4b200_stream_decode_to_device"][1][:5]
    # the CUDA-graph paragraph names both among the calls that refuse a capturing stream
    graphs = re.sub(r"\s+", " ", hdr[hdr.index("---- CUDA graphs"):hdr.index("int lz4b200_reserve(")])
    for name in CALLS:
        assert name[len("lz4b200_"):] in graphs, name


def test_without_a_device_both_calls_fail_and_write_nothing(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lz4net_b200 import native
    h = C.c_void_p()
    assert lib.lz4b200_create(C.byref(h), 0) == native.E_NODEVICE and not h.value
    src = np.frombuffer(b"\x00\x02ab", np.uint8).copy()                 # a one-chunk stream of two stored bytes
    dst = np.full(64, 0xEE, np.uint8)
    size = np.full(1, -7, np.int64)
    p = lambda a: a.ctypes.data                                                                 # noqa: E731
    calls = {
        CALLS[0]: (h, p(src), 4, 16, 0, p(dst), 64, p(size), None),
        CALLS[1]: (h, p(src), 4, p(dst), 64, p(size), None),
    }
    for name, args in calls.items():
        assert getattr(lib, name)(*args) < 0 and native.last_error(), name
        assert (dst == 0xEE).all() and size[0] == -7, name


class _NoContext:
    handle = None


def test_python_wrappers_refuse_host_tensors_that_are_not_page_locked(lib):
    """Each refusal is a TypeError raised before the library is called (the context here is no context at all)."""
    import torch
    from lz4net_b200 import batch
    pageable = torch.zeros(64, dtype=torch.uint8)
    size = torch.zeros(1, dtype=torch.int64)
    raw = torch.zeros(64, dtype=torch.uint8)
    nc = _NoContext()
    with pytest.raises(TypeError, match="dst: expected a page-locked CPU tensor"):
        batch.stream_encode_to_host_async(nc, raw, pageable, size)
    with pytest.raises(TypeError, match="wire: expected a page-locked CPU tensor"):
        batch.stream_decode_to_device_async(nc, pageable, 4, raw, size)
    with pytest.raises(TypeError, match="dst: expected a contiguous"):
        batch.stream_encode_to_host_async(nc, raw, np.zeros(64, np.uint8), size)             # dst: numpy, not a tensor
    with pytest.raises(TypeError, match="wire: expected a contiguous"):
        batch.stream_decode_to_device_async(nc, pageable[:2], 4, raw, size)                  # wire: shorter than n
    with pytest.raises(TypeError, match="dst: expected a contiguous"):
        batch.stream_encode_to_host_async(nc, raw, pageable.to(torch.int8), size)            # dst: not uint8


def test_cpp_mirror_methods_compile_against_the_header(tmp_path):
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c",
                           os.path.join(ROOT, "tests", "cpp", "async_stream_mirror.cpp"), "-o", str(tmp_path / "async_stream_mirror.o")])
