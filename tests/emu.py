"""ctypes driver for the CPU warp emulator (tests/simt_emu) -- TEST INFRASTRUCTURE ONLY.

It compiles the *kernel headers themselves* (lz4net_b200/csrc/*.cuh) with g++ in emulation mode so that the
warp-level algorithms can be checked against the oracle in a container without a GPU.  Nothing here is a product
code path: liblz4b200.so contains no CPU codec.

The library is built in a per-user temporary directory, keyed by the compiler flags and the contents of every source
and header it depends on, and installed with an atomic rename: the checkout may be read-only, and test processes that
start together never load a half-written file.
"""
from __future__ import annotations

import contextlib
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
_lib = None

HCW_FALLBACK = -2 ** 31

_P, _I, _U64 = C.c_void_p, C.c_int, C.c_uint64
_SIGNATURES = {                                                   # name: (restype, argtypes)
    "emu_decode": (None, [_I, _I, _I, _P, _P, _P, _P, _P, _U64]),
    "emu_decode_lpb": (None, [_I, _I, _I, _P, _P, _P, _P, _P, _U64]),
    "emu_encode": (None, [_I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _U64]),
    "emu_encode_hc": (_I, [_P, _I, _P, _I]),
    "emu_encode_hcw": (_I, [_P, _I, _P, _I, _U64, _I]),
    "emu_encode_hcw_window": (_I, [_P, _I, _P, _I, _U64]),
    "emu_measure": (None, [_I, _I, _P, _P, _P, _P, _U64]),
}


def build(source, defines=()):
    """Compiles simt_emu.cpp and the harness unit `source` with the extra -D flags `defines`; returns the library's path."""
    flags = ["-O2", "-g", "-shared", "-fPIC", "-std=c++17", "-DLZ4B200_SIMT_EMU", *defines]
    sources = [os.path.join(_DIR, "simt_emu.cpp"), source]
    deps = sources + [os.path.join(_DIR, "simt_emu.h")] + \
        sorted(os.path.join(_CSRC, f) for f in os.listdir(_CSRC) if f.endswith((".cuh", ".h")))
    h = hashlib.sha256(" ".join(flags).encode())
    for f in deps:
        with open(f, "rb") as fh:
            h.update(fh.read())
    out_dir = os.path.join(tempfile.gettempdir(), f"lz4b200_simt_emu_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, f"{os.path.splitext(os.path.basename(source))[0]}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call(["g++", *flags, "-I" + _DIR, "-I" + _CSRC, "-o", tmp] + sources)
        os.replace(tmp, so)
    return so


def lib():
    global _lib
    if _lib is None:
        l = C.CDLL(build(os.path.join(_DIR, "emu_harness.cpp")))
        for name, (restype, argtypes) in _SIGNATURES.items():
            getattr(l, name).restype = restype
            getattr(l, name).argtypes = argtypes
        _lib = l
    return _lib


def _bound(n):
    return n + n // 255 + 16


_libc = C.CDLL(None, use_errno=True)
_libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]


@contextlib.contextmanager
def _fenced(block, fence, pad):
    """Maps `block` next to a PROT_NONE page, `pad` readable bytes between them: behind its last byte (fence="behind")
    or in front of its first (fence="front").  At least a page stays readable on the other side.  Yields its address;
    the mapping lives, and the page stays fenced, until the with-block ends."""
    assert fence in ("behind", "front") and 0 <= pad < 4
    page = mmap.PAGESIZE
    n = len(block)
    npages = (pad + n + page - 1) // page + 1
    m = mmap.mmap(-1, (npages + 1) * page)
    base = C.addressof(C.c_char.from_buffer(m))
    guard, start = (base + npages * page, npages * page - pad - n) if fence == "behind" else (base, page + pad)
    m[start:start + n] = block
    assert _libc.mprotect(guard, page, 0) == 0                      # PROT_NONE
    try:
        yield base + start
    finally:
        assert _libc.mprotect(guard, page, mmap.PROT_READ | mmap.PROT_WRITE) == 0


@contextlib.contextmanager
def _staged(blocks, skew=0, fence=None, pad=0):
    """Yields one source address per block.  Each block lies `skew` bytes into its own zero-filled buffer with 64 bytes
    behind it; or, with `fence`, the one block lies `pad` bytes from a PROT_NONE page (see _fenced): a read of any
    word that holds no input byte kills the process with SIGSEGV."""
    if fence is not None:
        assert len(blocks) == 1 and skew == 0
        with _fenced(blocks[0], fence, pad) as p:
            yield [p]
        return
    bufs = []
    for b in blocks:
        a = np.zeros(skew + len(b) + 64, np.uint8)
        a[skew:skew + len(b)] = np.frombuffer(b, np.uint8)
        bufs.append(a)
    yield [a.ctypes.data + skew for a in bufs]


class _Slots:
    """Destination slots of `cap` bytes each, behind a red zone of 32 + skew bytes and in front of one of 64, all 0xCD."""

    def __init__(self, caps, skew=0):
        self.caps = [max(c, 0) for c in caps]
        self.lo = 32 + skew
        self.bufs = [np.full(c + 96 + skew, 0xCD, np.uint8) for c in self.caps]
        self.ptrs = [a.ctypes.data + self.lo for a in self.bufs]

    def take(self, lengths, who):
        """Asserts that no red zone changed; returns the first `length` bytes of each slot."""
        lo = self.lo
        for d, c in zip(self.bufs, self.caps):
            assert (d[:lo] == 0xCD).all() and (d[lo + c:] == 0xCD).all(), f"{who} wrote outside [dst, dst+cap)"
        return [d[lo:lo + max(r, 0)].tobytes() for d, r in zip(self.bufs, lengths)]


def _ptrs(addrs):
    return (C.c_void_p * len(addrs))(*addrs)


def decode(blocks, caps, lanes=32, known=True, sched_seed=1, src_skew=0, dst_skew=0, fence=None, pad=0):
    """blocks: list of bytes (compressed); caps: list of int. Returns (results, outputs).  src_skew shifts the
    compressed bytes inside their buffer to exercise unaligned stream starts; fence / pad: see _staged."""
    n = len(blocks)
    isz = np.array([len(b) for b in blocks], np.int32)
    cps = np.array(caps, np.int32)
    res = np.zeros(n, np.int32)
    out = _Slots(caps, dst_skew)
    with _staged(blocks, src_skew, fence, pad) as src:
        args = (int(known), n, _ptrs(src), isz.ctypes.data, _ptrs(out.ptrs), cps.ctypes.data, res.ctypes.data, sched_seed)
        if lanes in (1, 2):      # lane-per-block decoder (1: the kernel's geometry, 2: larger rings / 64-byte runs / one sequence per iteration)
            lib().emu_decode_lpb(lanes - 1, *args)
        else:
            lib().emu_decode(lanes, *args)
    return res.tolist(), out.take(caps, "decoder")


def encode(blocks, caps=None, sched_seed=1, src_skew=0, dst_skew=0, variant=2, tune=(12, 8, 24), fence=None, pad=0):
    """variant: how the encoder finds same-hash lanes inside a round (1 always exact votes, 2 optimistic = the default);
    tune: (lane_copy_max, probe_max, wide_min), EncTune's defaults unless given.  fence / pad: see _staged."""
    n = len(blocks)
    if caps is None:
        caps = [_bound(len(b)) for b in blocks]
    ns = np.array([len(b) for b in blocks], np.int32)
    cps = np.array(caps, np.int32)
    res = np.zeros(n, np.int32)
    out = _Slots(caps, dst_skew)
    with _staged(blocks, src_skew, fence, pad) as src:
        lib().emu_encode(variant, *tune, n, _ptrs(src), ns.ctypes.data, _ptrs(out.ptrs), cps.ctypes.data, res.ctypes.data,
                         sched_seed)
    return res.tolist(), out.take(res.tolist(), "encoder")


def _encode_one(entry, who, block, cap, src_skew, dst_skew, fence, *args):
    """One block through a single-block encoder entry point.  Returns (result, bytes)."""
    n = len(block)
    if cap is None:
        cap = _bound(n)
    out = _Slots([cap], dst_skew)
    with _staged([block], src_skew, fence) as (src,):
        r = getattr(lib(), entry)(src, n, out.ptrs[0], cap, *args)
    return r, out.take([r], who)[0]


def encode_hc(block, cap=None, src_skew=0):
    return _encode_one("emu_encode_hc", "HC encoder", block, cap, src_skew, 0, None)


def encode_hcw(block, cap=None, src_skew=0, dst_skew=0, sched_seed=1, smem=True):
    """The warp-per-block HC encoder (lz4hc_warp.cuh).  Returns (result, bytes); result == HCW_FALLBACK when the kernel hands
    the block to the thread-per-block one.  smem: block staged in shared memory; else read through the read-only path."""
    return _encode_one("emu_encode_hcw", "HC warp encoder", block, cap, src_skew, dst_skew, None, sched_seed, int(smem))


def encode_hcw_window(block, cap=None, src_skew=0, dst_skew=0, sched_seed=1, fence=None):
    """The windowed HC warp encoder (lz4hc_window.cuh, blocks above 64 KiB).  Returns (result, bytes); result ==
    HCW_FALLBACK when the kernel hands the block to the thread-per-block one.  fence: see _staged."""
    return _encode_one("emu_encode_hcw_window", "window encoder", block, cap, src_skew, dst_skew, fence, sched_seed)


def measure(blocks, caps=None, known=False, sched_seed=1, src_skew=0, fence=None):
    """The measure pass (lz4_measure.cuh) over compressed blocks; caps=None = no limit (INT32_MAX per block).  src_skew
    shifts each block inside its buffer (unaligned stream starts); fence: see _staged.  Returns the per-block results."""
    n = len(blocks)
    isz = np.array([len(b) for b in blocks], np.int32)
    cps = None if caps is None else np.array(caps, np.int32)
    res = np.zeros(n, np.int32)
    with _staged(blocks, src_skew, fence) as src:
        lib().emu_measure(int(known), n, _ptrs(src), isz.ctypes.data, None if cps is None else cps.ctypes.data,
                          res.ctypes.data, sched_seed)
    return res.tolist()
