"""CPU-only: the C-ABI library builds for sm_90a (H100), loads, and exports exactly what include/lz4b200.h declares.
No compute calls here (no GPU in this container); the product must refuse to run without a device."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from lz4net_b200 import build, native
    build.build()
    return native.lib()


def test_header_and_binding_agree(lib):
    from lz4net_b200 import native
    hdr = open(os.path.join(ROOT, "include", "lz4b200.h")).read()
    declared = set(re.findall(r"\b(lz4b200_[a-zA-Z0-9_]+)\s*\(", hdr)) - {"lz4b200_ctx"}
    assert declared == set(native.SIGNATURES), declared ^ set(native.SIGNATURES)
    for name in declared:
        assert hasattr(lib, name), name


def test_constants(lib):
    assert lib.lz4b200_version() == 100
    assert lib.lz4b200_compress_bound(65536) == 65809            # src/LZ4/LZ4Codec.cs:313-316
    assert lib.lz4b200_compress_bound(0) == 16
    assert lib.lz4b200_stream_bound(65536 * 3 + 1, 65536) == 65536 * 3 + 1 + 4 * (1 + 2 * 3)


def test_no_cpu_fallback(lib):
    """Without a device the library reports failure instead of computing on the host."""
    import ctypes as C
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from lz4net_b200 import native
    assert lib.lz4b200_device_count() == 0
    h = C.c_void_p()
    assert lib.lz4b200_create(C.byref(h), 0) == native.E_NODEVICE
    src = C.create_string_buffer(b"a" * 64); dst = C.create_string_buffer(128)
    assert lib.lz4b200_compress_limitedOutput(src, dst, 64, 128) == 0        # encoder failure value
    assert lib.lz4b200_uncompress(src, dst, 64, 128) < 0                     # decoder error value


def test_only_sm90a_code_in_binary():
    import subprocess
    from lz4net_b200 import native
    out = subprocess.run(["cuobjdump", "-lelf", native.SO_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs
    sass = subprocess.run(["cuobjdump", "-sass", native.SO_PATH], capture_output=True, text=True).stdout
    assert "UBLKCP" in sass and "SYNCS" in sass and "MATCH.ANY" in sass     # TMA bulk copy + mbarrier + warp match


def test_framing_helpers_without_gpu(lib):
    """Header walking is host code: sizes and corruption checks work without a device (LZ4Stream.cs:274-293)."""
    import numpy as np
    from lz4net_b200 import native

    def size(b):
        a = np.frombuffer(b + b"\0", np.uint8)
        return lib.lz4b200_stream_decoded_size(a.ctypes.data, len(b))
    assert size(b"") == 0
    assert size(bytes([0, 5]) + b"hello") == 5                                # stored chunk
    assert size(bytes([0, 5]) + b"hell") == native.E_FORMAT                   # truncated payload
    assert size(bytes([1, 5, 6]) + b"xxxxxx") == native.E_FORMAT              # compLen > rawLen
    assert size(bytes([0x80])) == native.E_FORMAT                             # truncated varint
    assert size(bytes([5, 100, 3]) + b"abc") == native.E_FORMAT               # passes != 0
    a = np.frombuffer(bytes([100, 0, 0, 0, 3, 0, 0, 0]) + b"abc" + b"\0", np.uint8)
    assert lib.lz4b200_unwrap_size(a.ctypes.data, 11) == 100
    assert lib.lz4b200_unwrap_size(a.ctypes.data, 10) == native.E_FORMAT
