"""ctypes driver for the windowed LZ4HC warp encoder (lz4net_b200/csrc/lz4hc_window.cuh, blocks above 64 KiB) on the CPU warp
emulator -- TEST INFRASTRUCTURE ONLY.

The kernel header itself is compiled with g++ in emulation mode (tests/simt_emu/emu_hcw_window.cpp + simt_emu.cpp).  The
library is built in a per-user temporary directory, keyed by the sources' contents: the checkout itself may be read-only.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import mmap
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_DIR = os.path.join(_HERE, "simt_emu")
_CSRC = os.path.join(_ROOT, "lz4net_b200", "csrc")
_SOURCES = [os.path.join(_DIR, f) for f in ("simt_emu.cpp", "emu_hcw_window.cpp")]
_DEPS = _SOURCES + [os.path.join(_DIR, "simt_emu.h")] + \
    [os.path.join(_CSRC, f) for f in ("lz4hc_window.cuh", "lz4hc_warp.cuh", "lz4_copy.cuh", "simt.cuh")]
_lib = None

HCW_FALLBACK = -2 ** 31


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for f in _DEPS:
            with open(f, "rb") as fh:
                h.update(fh.read())
        out_dir = os.path.join(tempfile.gettempdir(), f"lz4b200_emu_hcw_window_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        so = os.path.join(out_dir, f"libemu_hcw_window_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["g++", "-O2", "-g", "-shared", "-fPIC", "-std=c++17", "-DLZ4B200_SIMT_EMU",
                                   "-I" + _DIR, "-I" + _CSRC, "-o", tmp] + _SOURCES)
            os.replace(tmp, so)
        _lib = C.CDLL(so)
        _lib.emu_encode_hcw_window.restype = C.c_int
        _lib.emu_encode_hcw_window.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_uint64]
    return _lib


def encode(block, cap=None, src_skew=0, dst_skew=0, sched_seed=1):
    """One block through the windowed kernel.  Returns (result, bytes); result == HCW_FALLBACK when the kernel hands the
    block to the thread-per-block one.  Asserts that nothing outside [dst, dst + cap) was written."""
    n = len(block)
    if cap is None:
        cap = n + n // 255 + 16
    a = np.zeros(src_skew + n + 64, np.uint8)
    a[src_skew:src_skew + n] = np.frombuffer(block, np.uint8)
    lo = 32 + dst_skew
    d = np.full(max(cap, 0) + 96 + dst_skew, 0xCD, np.uint8)
    r = lib().emu_encode_hcw_window(a.ctypes.data + src_skew, n, d.ctypes.data + lo, cap, sched_seed)
    assert (d[:lo] == 0xCD).all() and (d[lo + max(cap, 0):] == 0xCD).all(), "window encoder wrote outside [dst, dst+cap)"
    return int(r), d[lo:lo + max(r, 0)].tobytes()


def encode_fenced(block, behind=True):
    """Encode one block with a PROT_NONE page directly behind its last byte (behind=True) or directly in front of its first
    byte (behind=False): a read of any word that holds no input byte kills the process with SIGSEGV.  Returns (result, bytes)."""
    page = mmap.PAGESIZE
    n = len(block)
    npages = (n + page - 1) // page + 1
    m = mmap.mmap(-1, (npages + 2) * page)
    base = C.addressof(C.c_char.from_buffer(m))
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    fence = base + (npages + 1) * page if behind else base
    start = (npages + 1) * page - n if behind else page
    m[start:start + n] = block
    assert libc.mprotect(fence, page, 0) == 0
    cap = n + n // 255 + 16
    d = np.full(cap + 96, 0xCD, np.uint8)
    try:
        r = lib().emu_encode_hcw_window(base + start, n, d.ctypes.data + 32, cap, 1)
    finally:
        assert libc.mprotect(fence, page, 3) == 0
    return int(r), d[32:32 + max(r, 0)].tobytes()
