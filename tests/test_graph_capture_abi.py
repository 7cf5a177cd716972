"""CPU-only: lz4b200_reserve is exported, declared and bound, and refuses a null context or a negative block count before it
touches a device (so it does so on a machine without one)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from lz4net_b200 import build, native
    build.build()
    return native.lib()


def test_reserve_is_declared_and_bound(lib):
    from lz4net_b200 import native
    hdr = open(os.path.join(ROOT, "include", "lz4b200.h")).read()
    assert re.search(r"\bint\s+lz4b200_reserve\s*\(\s*lz4b200_ctx\s*\*\s*ctx,\s*int32_t max_blocks,\s*int high_compression\)", hdr)
    assert native.SIGNATURES["lz4b200_reserve"] == (C.c_int, [C.c_void_p, C.c_int32, C.c_int])
    assert hasattr(lib, "lz4b200_reserve")


def test_reserve_null_context(lib):
    from lz4net_b200 import native
    for hc in (0, 1):
        assert lib.lz4b200_reserve(None, 16, hc) == native.E_ARG
        assert "null context" in native.last_error()


def test_reserve_negative_block_count(lib):
    """A non-null handle that is never dereferenced: the count is checked first."""
    from lz4net_b200 import native
    bogus = C.c_void_p(1)
    assert lib.lz4b200_reserve(bogus, -1, 0) == native.E_ARG
    assert "negative" in native.last_error()
    assert lib.lz4b200_reserve(bogus, -(1 << 31), 1) == native.E_ARG


def test_context_reserve_raises_without_a_context(lib):
    from lz4net_b200 import native
    from lz4net_b200.codec import Context
    ctx = Context.__new__(Context)
    ctx._h = C.c_void_p()
    with pytest.raises(native.Lz4B200Error, match="status -1"):
        ctx.reserve(8, hc=True)
