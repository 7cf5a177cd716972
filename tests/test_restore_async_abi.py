"""CPU-only: the asynchronous decode and Unwrap from device-written offsets (lz4b200_decode_batch_to_device_at_async,
lz4b200_unwrap_batch_to_device_at_async) are declared, bound and exported; without a device they fail and write nothing;
the Python wrappers refuse host tensors that are not page-locked, for the source and for src_off, before the library sees
them; the C++ mirror's methods compile against the header."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# each call and the host-offset form it restates with (src_cap, device-read src_off) in place of (src_off, src_len)
PAIRS = {
    "lz4b200_decode_batch_to_device_at_async": "lz4b200_decode_batch_to_device_async",
    "lz4b200_unwrap_batch_to_device_at_async": "lz4b200_unwrap_batch_to_device_async",
}


@pytest.fixture(scope="module")
def lib():
    from lz4net_b200 import build, native
    build.build()
    return native.lib()


def test_symbols_are_declared_bound_and_exported(lib):
    from lz4net_b200 import native
    hdr = open(os.path.join(ROOT, "include", "lz4b200.h")).read()
    for name, host_form in PAIRS.items():
        assert re.search(r"\bint\s+%s\s*\(" % name, hdr), name
        assert hasattr(lib, name), name
        res, args = native.SIGNATURES[name]
        hres, hargs = native.SIGNATURES[host_form]
        # ctx, src | src_cap (int64), src_off | the rest as in the host-offset form
        assert res == hres and args[:2] == hargs[:2] and args[2] == C.c_int64 and args[3:] == hargs[3:], name
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
    so, dof, cap = np.array([0, 10], np.int64), np.zeros(1, np.int64), np.array([64], np.int32)
    dst = np.full(64, 0xEE, np.uint8)
    out = np.full(1, 12345, np.int32)
    p = lambda a: a.ctypes.data                                                                 # noqa: E731
    calls = {
        "lz4b200_decode_batch_to_device_at_async": (h, p(src), 10, p(so), p(dst), p(dof), p(cap), p(out), 1, 1, None),
        "lz4b200_unwrap_batch_to_device_at_async": (h, p(src), 10, p(so), p(dst), p(dof), p(cap), p(out), 1, None),
    }
    for name, args in calls.items():
        assert getattr(lib, name)(*args) < 0 and native.last_error(), name
        assert (dst == 0xEE).all() and out[0] == 12345 and list(so) == [0, 10], name


class _NoContext:
    handle = None


def test_python_wrappers_refuse_host_tensors_that_are_not_page_locked(lib):
    """Each refusal is a TypeError (or, for src_cap, a ValueError) raised before the library is called (the context here is
    no context at all).  The source is checked first, so the refusals of src_off need a page-locked source, which only a
    machine with a GPU can allocate."""
    import torch
    from lz4net_b200 import batch
    n = 2
    dof, cap = np.zeros(n, np.int64), np.full(n, 32, np.int32)
    pageable = torch.zeros(64, dtype=torch.uint8)
    off, out = torch.zeros(n + 1, dtype=torch.int64), torch.zeros(n, dtype=torch.int32)
    raw = torch.zeros(64, dtype=torch.uint8)
    nc = _NoContext()
    for fn, what in ((batch.decode_from_host_at_async, "comp"), (batch.unwrap_to_device_at_async, "packets")):
        with pytest.raises(TypeError, match=f"{what}: expected a page-locked CPU tensor"):
            fn(nc, pageable, 64, off, raw, dof, cap, out)
        with pytest.raises(TypeError):
            fn(nc, np.zeros(64, np.uint8), 64, off, raw, dof, cap, out)                    # source: numpy, not a tensor
        if torch.cuda.is_available():
            pinned = torch.zeros(64, dtype=torch.uint8).pin_memory()
            with pytest.raises(TypeError, match="src_off: expected a page-locked CPU tensor"):
                fn(nc, pinned, 64, off, raw, dof, cap, out)                                 # src_off: pageable
            with pytest.raises(TypeError, match="src_off: expected a contiguous"):
                fn(nc, pinned, 64, off.to(torch.int32).pin_memory(), raw, dof, cap, out)     # src_off: not int64
            with pytest.raises(ValueError, match="src_cap"):
                fn(nc, pinned, 65, off.pin_memory(), raw, dof, cap, out)                     # beyond the source


def test_cpp_mirror_methods_compile_against_the_header(tmp_path):
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-c",
                           os.path.join(ROOT, "tests", "cpp", "async_restore_mirror.cpp"), "-o", str(tmp_path / "m.o")])
