"""CPU-only: the LZ4Stream decode from a device-written size (lz4b200_stream_decode_to_device_at_async) is declared, bound
and exported; without a device it fails and writes nothing; the Python wrapper refuses host tensors that are not
page-locked and a src_cap beyond the source before the library sees them; the C++ mirror's method compiles against the
header."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "lz4b200_stream_decode_to_device_at_async"


@pytest.fixture(scope="module")
def lib():
    from lz4net_b200 import build, native
    build.build()
    return native.lib()


def test_symbol_is_declared_bound_and_exported(lib):
    from lz4net_b200 import native
    hdr = open(os.path.join(ROOT, "include", "lz4b200.h")).read()
    assert re.search(r"\bint\s+%s\s*\(" % NAME, hdr)
    assert hasattr(lib, NAME)
    # ctx, src, src_cap, src_size, block_size, dst, dst_cap, out_size, stream
    assert native.SIGNATURES[NAME] == (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_int64,
                                                 C.c_void_p, C.c_void_p])
    graphs = hdr[hdr.index("---- CUDA graphs"):hdr.index("int lz4b200_reserve(")]
    assert NAME[len("lz4b200_"):] in re.sub(r"\s+", " ", graphs)


def test_without_a_device_the_call_fails_and_writes_nothing(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lz4net_b200 import native
    h = C.c_void_p()
    assert lib.lz4b200_create(C.byref(h), 0) == native.E_NODEVICE and not h.value
    src = np.frombuffer(b"\x00\x02ab" + bytes(12), np.uint8).copy()
    size, out = np.array([4], np.int64), np.full(1, 12345, np.int64)
    dst = np.full(64, 0xEE, np.uint8)
    p = lambda a: a.ctypes.data                                                                 # noqa: E731
    for ctx in (h, None):
        assert lib.lz4b200_stream_decode_to_device_at_async(ctx, p(src), 4, p(size), 16, p(dst), 64, p(out), None) < 0
        assert native.last_error()
    assert (dst == 0xEE).all() and out[0] == 12345 and size[0] == 4


class _NoContext:
    handle = None


def test_python_wrapper_refuses_host_tensors_that_are_not_page_locked(lib):
    """Each refusal is raised before the library is called (the context here is no context at all).  The source is checked
    first, so the refusals of src_size and out_size need a page-locked source, which only a machine with a GPU allocates."""
    import torch
    from lz4net_b200 import batch
    pageable = torch.zeros(64, dtype=torch.uint8)
    cell = torch.zeros(1, dtype=torch.int64)
    out = torch.zeros(64, dtype=torch.uint8)
    nc = _NoContext()
    with pytest.raises(TypeError, match="wire: expected a page-locked CPU tensor"):
        batch.stream_decode_to_device_at_async(nc, pageable, 64, cell, out, cell)
    with pytest.raises(TypeError):
        batch.stream_decode_to_device_at_async(nc, np.zeros(64, np.uint8), 64, cell, out, cell)      # numpy, not a tensor
    if torch.cuda.is_available():
        pinned = torch.zeros(64, dtype=torch.uint8).pin_memory()
        with pytest.raises(ValueError, match="src_cap"):
            batch.stream_decode_to_device_at_async(nc, pinned, 65, cell.pin_memory(), out, cell.pin_memory())
        with pytest.raises(TypeError, match="src_size: expected a page-locked CPU tensor"):
            batch.stream_decode_to_device_at_async(nc, pinned, 64, cell, out, cell.pin_memory())
        with pytest.raises(TypeError, match="src_size: expected a contiguous"):
            batch.stream_decode_to_device_at_async(nc, pinned, 64, cell.to(torch.int32).pin_memory(), out, cell.pin_memory())
        with pytest.raises(TypeError, match="out_size: expected a page-locked CPU tensor"):
            batch.stream_decode_to_device_at_async(nc, pinned, 64, cell.pin_memory(), out, cell)
        with pytest.raises(TypeError, match="expected a torch CUDA tensor"):
            batch.stream_decode_to_device_at_async(nc, pinned, 64, cell.pin_memory(), out, cell.pin_memory())   # out on the CPU


def test_cpp_mirror_method_compiles_against_the_header(tmp_path):
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c",
                           os.path.join(ROOT, "tests", "cpp", "async_stream_restore_mirror.cpp"), "-o", str(tmp_path / "m.o")])
