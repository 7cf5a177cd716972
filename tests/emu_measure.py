"""ctypes driver for the measure pass (lz4net_b200/csrc/lz4_measure.cuh) on the CPU warp emulator -- TEST INFRASTRUCTURE ONLY.

The kernel header itself is compiled with g++ in emulation mode (tests/simt_emu/emu_measure.cpp + simt_emu.cpp), so that
its verdicts can be checked against the oracle without a GPU.  The library is built in a per-user temporary directory,
keyed by the sources' contents: the checkout itself may be read-only.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_DIR = os.path.join(_HERE, "simt_emu")
_CSRC = os.path.join(_ROOT, "lz4net_b200", "csrc")
_SOURCES = [os.path.join(_DIR, f) for f in ("simt_emu.cpp", "emu_measure.cpp")]
_DEPS = _SOURCES + [os.path.join(_DIR, "simt_emu.h"), os.path.join(_CSRC, "lz4_measure.cuh"), os.path.join(_CSRC, "simt.cuh")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for f in _DEPS:
            with open(f, "rb") as fh:
                h.update(fh.read())
        out_dir = os.path.join(tempfile.gettempdir(), f"lz4b200_emu_measure_{os.getuid()}")
        os.makedirs(out_dir, exist_ok=True)
        so = os.path.join(out_dir, f"libemu_measure_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["g++", "-O2", "-g", "-shared", "-fPIC", "-std=c++17", "-DLZ4B200_SIMT_EMU",
                                   "-I" + _DIR, "-I" + _CSRC, "-o", tmp] + _SOURCES)
            os.replace(tmp, so)
        _lib = C.CDLL(so)
    return _lib


def _run(srcs, isz, caps, known, sched_seed):
    n = len(srcs)
    cps = None if caps is None else np.array(caps, np.int32)
    res = np.zeros(n, np.int32)
    sp = (C.c_void_p * n)(*srcs)
    lib().emu_measure(int(known), n, sp, isz.ctypes.data_as(C.c_void_p), None if cps is None else cps.ctypes.data_as(C.c_void_p),
                      res.ctypes.data_as(C.c_void_p), C.c_uint64(sched_seed))
    return res.tolist()


def measure(blocks, caps=None, known=False, sched_seed=1, src_skew=0):
    """The measure pass over compressed blocks; caps=None = no limit (INT32_MAX per block).  src_skew shifts each block
    inside its buffer (unaligned stream starts).  Returns the per-block results."""
    bufs = []
    for b in blocks:
        a = np.zeros(src_skew + len(b) + 64, np.uint8)
        a[src_skew:src_skew + len(b)] = np.frombuffer(b, np.uint8)
        bufs.append(a)
    isz = np.array([len(b) for b in blocks], np.int32)
    return _run([a.ctypes.data + src_skew for a in bufs], isz, caps, known, sched_seed)


def measure_guarded(block, cap=None, known=False):
    """Measure one block that ends on a 16-byte boundary which is also the end of a readable page (the next page is
    PROT_NONE): a read of any unit past the block's last one kills the process with SIGSEGV."""
    import mmap
    page = mmap.PAGESIZE
    n = len(block)
    npages = (n + page - 1) // page + 1
    m = mmap.mmap(-1, (npages + 1) * page)
    base = C.addressof(C.c_char.from_buffer(m))
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    assert libc.mprotect(base + npages * page, page, 0) == 0
    start = npages * page - n
    m[start:start + n] = block
    r = _run([base + start], np.array([n], np.int32), None if cap is None else [cap], known, 1)[0]
    assert libc.mprotect(base + npages * page, page, 3) == 0
    return int(r)
