"""CPU-only: the asynchronous offload calls (lz4b200_encode_batch_packed_from_device_async,
lz4b200_decode_batch_to_device_async) are declared, bound and exported; without a device they fail and write nothing; the
Python wrappers refuse host tensors that are not page-locked before the library sees them."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENCODE = "lz4b200_encode_batch_packed_from_device_async"
DECODE = "lz4b200_decode_batch_to_device_async"


@pytest.fixture(scope="module")
def lib():
    from lz4net_b200 import build, native
    build.build()
    return native.lib()


def test_symbols_are_declared_bound_and_exported_like_the_synchronous_calls(lib):
    from lz4net_b200 import native
    hdr = open(os.path.join(ROOT, "include", "lz4b200.h")).read()
    for name in (ENCODE, DECODE):
        assert re.search(r"\bint\s+%s\s*\(" % name, hdr)
        assert hasattr(lib, name)
    # the encode takes the parameter list of its synchronous form; the decode that of decode_batch without `mem`
    assert native.SIGNATURES[ENCODE] == native.SIGNATURES["lz4b200_encode_batch_packed_from_device"]
    res, args = native.SIGNATURES["lz4b200_decode_batch"]
    assert native.SIGNATURES[DECODE] == (res, args[:10] + args[11:])


def test_without_a_device_both_calls_fail_and_write_nothing(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lz4net_b200 import native
    h = C.c_void_p()
    assert lib.lz4b200_create(C.byref(h), 0) == native.E_NODEVICE and not h.value
    src = np.frombuffer(b"\x10a" + bytes(16), np.uint8).copy()
    so, sl, cap = np.zeros(1, np.int64), np.array([2], np.int32), np.array([64], np.int32)
    dst = np.full(64, 0xEE, np.uint8)
    off, out = np.full(2, -7, np.int64), np.full(1, 12345, np.int32)
    rc = getattr(lib, ENCODE)(h, src.ctypes.data, so.ctypes.data, sl.ctypes.data, cap.ctypes.data, dst.ctypes.data, 64,
                              off.ctypes.data, out.ctypes.data, 1, native.MODE_FAST, None)
    assert rc < 0 and native.last_error()
    assert (dst == 0xEE).all() and (off == -7).all() and out[0] == 12345
    rc = getattr(lib, DECODE)(h, src.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data, so.ctypes.data, cap.ctypes.data,
                              out.ctypes.data, 1, 1, None)
    assert rc < 0 and native.last_error()
    assert (dst == 0xEE).all() and out[0] == 12345


class _NoContext:
    handle = None


def test_python_wrappers_refuse_host_tensors_that_are_not_page_locked(lib):
    """Each refusal is a TypeError raised before the library is called (the context here is no context at all)."""
    import torch
    from lz4net_b200 import batch
    n = 2
    so, sl, cap = np.zeros(n, np.int64), np.ones(n, np.int32), np.full(n, 32, np.int32)
    pageable = torch.zeros(64, dtype=torch.uint8)
    off, out = torch.zeros(n + 1, dtype=torch.int64), torch.zeros(n, dtype=torch.int32)
    raw = torch.zeros(64, dtype=torch.uint8)
    enc = lambda *a: batch.encode_to_host_packed_async(_NoContext(), raw, so, sl, cap, *a)          # noqa: E731
    dec = lambda *a: batch.decode_from_host_async(_NoContext(), *a)                                # noqa: E731
    with pytest.raises(TypeError, match="dst: expected a page-locked CPU tensor"):
        enc(pageable, off, out)
    with pytest.raises(TypeError, match="comp: expected a page-locked CPU tensor"):
        dec(pageable, so, sl, raw, so, cap, out)
    with pytest.raises(TypeError):
        dec(np.zeros(64, np.uint8), so, sl, raw, so, cap, out)                                     # comp: numpy, not a tensor
    with pytest.raises(TypeError, match="dst: expected a contiguous"):
        enc(pageable.to(torch.int8), off, out)                                                     # dst: not uint8
