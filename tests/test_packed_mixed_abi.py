"""CPU-only: lz4b200_decode_batch_packed_to_device is exported, declared and bound; it computes nothing without a device;
the Python wrappers refuse arguments the library would misread before they reach it."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "lz4b200_decode_batch_packed_to_device"


@pytest.fixture(scope="module")
def lib():
    from lz4net_b200 import build, native
    build.build()
    return native.lib()


def test_symbol_is_exported_declared_and_bound_like_the_device_call(lib):
    from lz4net_b200 import native
    hdr = open(os.path.join(ROOT, "include", "lz4b200.h")).read()
    assert re.search(r"\bint\s+%s\s*\(" % NAME, hdr)
    assert hasattr(lib, NAME)
    assert native.SIGNATURES[NAME] == native.SIGNATURES["lz4b200_decode_batch_packed"]       # the same parameter list


def test_no_cpu_fallback(lib):
    """Without a device there is no context to call it with, and without a context it reports failure and writes nothing."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lz4net_b200 import native
    h = C.c_void_p()
    assert lib.lz4b200_create(C.byref(h), 0) == native.E_NODEVICE and not h.value
    src = np.frombuffer(b"\x10a" + bytes(16), np.uint8).copy()                                # a well-formed block: one literal
    so, sl = np.zeros(1, np.int64), np.array([2], np.int32)
    dst = np.full(64, 0xEE, np.uint8)
    off, out = np.full(2, -7, np.int64), np.full(1, 12345, np.int32)
    rc = getattr(lib, NAME)(h, src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data, 64, off.ctypes.data,
                            out.ctypes.data, 1, None)
    assert rc < 0 and native.last_error()
    assert (dst == 0xEE).all() and (off == -7).all() and out[0] == 12345


class _NoContext:
    handle = None


def test_python_wrapper_checks_its_arrays_before_the_call(lib):
    import torch
    from lz4net_b200 import batch
    n = 3
    comp = np.zeros(64, np.uint8)
    so, sl = np.zeros(n, np.int64), np.zeros(n, np.int32)
    off, out = np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
    host_out = torch.zeros(64, dtype=torch.uint8)
    call = lambda *a: batch.decode_from_host_packed(_NoContext(), *a)                         # noqa: E731
    with pytest.raises(TypeError):
        call(comp.astype(np.int8), so, sl, host_out, off, out)                                # comp: not uint8
    with pytest.raises(TypeError):
        call(comp, so.astype(np.int32), sl, host_out, off, out)                               # src_off: not int64
    with pytest.raises(TypeError):
        call(comp, so, sl[:2], host_out, off, out)                                            # src_len: too short
    with pytest.raises(TypeError, match="int64 array of at least 4"):
        call(comp, so, sl, host_out, off[:n], out)                                            # out_off: n entries, not n + 1
    with pytest.raises(TypeError, match="int32 array of at least 3"):
        call(comp, so, sl, host_out, off, out.astype(np.int64))                               # out_len: not int32
    with pytest.raises(TypeError):
        call(comp[::2], so, sl, host_out, off, out)                                           # comp: not contiguous
    with pytest.raises(TypeError, match="CUDA tensor"):
        call(comp, so, sl, host_out, off, out)                                                # out: not device memory
    with pytest.raises(TypeError, match="CUDA tensor"):
        call(comp, so, sl, np.zeros(64, np.uint8), off, out)
