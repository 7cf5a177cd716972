"""CPU oracle for the LZ4 r93 block codec -- TEST INFRASTRUCTURE ONLY.

Two interchangeable implementations, both loaded through ctypes:

* ``port``  -- ``oracle/liblz4_oracle.so``: this repo's own plain-C restatement (``lz4_oracle.c``).
* ``ref``   -- ``oracle/_ref/liblz4net_ref.so``: the reference's ``original/lz4.c`` + ``original/lz4hc.c``
  compiled in place from the lz4net checkout named by ``$LZ4NET_REFERENCE`` by ``oracle/Makefile`` with lz4net's 64-bit shim flags
  (``src/adapters/cpp/lz4_64.h:5-9``).  lz4net's ConformanceTests assert this code byte-identical to every
  C# codec flavour (``src/LZ4.Tests/ConformanceTests.cs:59-68,125-132``), which is what makes it a valid
  stand-in for ``LZ4Codec.Encode`` bytes.  Optional: the tests read what it produced from ``tests/golden/``
  (``tests/golden/make_golden.py``), so they run without a lz4net checkout.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import this module.
The product package ``lz4net_b200`` never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_SO = os.path.join(_HERE, "liblz4_oracle.so")
_REF_SO = os.path.join(_HERE, "_ref", "liblz4net_ref.so")
REF_ENV = "LZ4NET_REFERENCE"                  # a MiloszKrajewski/lz4net checkout (only make_golden.py needs one)

_port = None
_ref = None


def build(force: bool = False) -> None:
    """Compile the port (always possible: gcc only) and, where $LZ4NET_REFERENCE names a lz4net checkout, oracle/_ref."""
    if force or not os.path.exists(_PORT_SO) or \
            os.path.getmtime(_PORT_SO) < max(os.path.getmtime(os.path.join(_HERE, f))
                                             for f in ("lz4_oracle.c", "lz4_oracle.h", "oracle_mt.c")):
        subprocess.check_call(["make", "-C", _HERE, "liblz4_oracle.so"], stdout=subprocess.DEVNULL)
    ref_dir = os.environ.get(REF_ENV, "")
    if ref_dir and os.path.exists(os.path.join(ref_dir, "original", "lz4.c")) and (force or not os.path.exists(_REF_SO)):
        subprocess.check_call(["make", "-C", _HERE, "ref", "REF=" + os.path.abspath(ref_dir)], stdout=subprocess.DEVNULL)


def _u8p(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint8))


def port():
    global _port
    if _port is None:
        build()
        lib = C.CDLL(_PORT_SO)
        u8p = C.POINTER(C.c_uint8)
        lib.lz4o_bound.argtypes = [C.c_int]
        lib.lz4o_encode.argtypes = [u8p, C.c_int, u8p, C.c_int]
        lib.lz4o_encode_hc.argtypes = [u8p, C.c_int, u8p, C.c_int]
        lib.lz4o_decode_known.argtypes = [u8p, C.c_int, u8p, C.c_int]
        lib.lz4o_decode_unknown.argtypes = [u8p, C.c_int, u8p, C.c_int]
        lib.lz4o_mt_run.restype = C.c_double
        lib.lz4o_mt_run.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        _port = lib
    return _port


def have_ref() -> bool:
    if not os.path.exists(_REF_SO):
        try:
            build()
        except Exception:
            pass
    return os.path.exists(_REF_SO)


def ref():
    global _ref
    if _ref is None:
        if not have_ref():
            raise RuntimeError(f"oracle/_ref/liblz4net_ref.so is absent (set {REF_ENV} to a lz4net checkout to build it)")
        lib = C.CDLL(_REF_SO)
        cp = C.c_char_p
        for name in ("LZ4_compress_limitedOutput", "LZ4_compressHC_limitedOutput", "LZ4_uncompress_unknownOutputSize"):
            getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        lib.LZ4_uncompress.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        _ref = lib
    return _ref


def bound(n: int) -> int:
    return n + n // 255 + 16


def _as_u8(data) -> np.ndarray:
    a = np.frombuffer(data, dtype=np.uint8) if isinstance(data, (bytes, bytearray, memoryview)) else np.asarray(data, dtype=np.uint8)
    return np.ascontiguousarray(a)


def _encode(data, cap, hc: bool, impl: str):
    src = _as_u8(data)
    n = src.size
    if cap is None:
        cap = bound(n)
    # Guard band behind `cap`.  It must absorb a real r93 quirk: LZ4_encodeSequence's second limit check uses the
    # LITERAL length (original/lz4hc.c:541), so with a tight cap a long match's n/255 length bytes are written past
    # `cap` before a later check returns 0 (the fast encoder can likewise spill a few bytes on >64 KiB matches).
    dst = np.full(max(cap, 0) + n // 255 + 64, 0xA5, dtype=np.uint8)
    srcp = np.concatenate([src, np.zeros(16, np.uint8)])  # reads never pass n, pad only to give a valid pointer for n == 0
    if impl == "port":
        fn = port().lz4o_encode_hc if hc else port().lz4o_encode
        r = fn(_u8p(srcp), n, _u8p(dst), cap)
    else:
        fn = ref().LZ4_compressHC_limitedOutput if hc else ref().LZ4_compress_limitedOutput
        r = fn(srcp.ctypes.data, dst.ctypes.data, n, cap)
    return int(r), dst


def encode(data, cap=None, impl: str = "port"):
    """LZ4_compress_limitedOutput semantics: returns (ret, bytes) with ret == 0 on failure."""
    r, dst = _encode(data, cap, False, impl)
    return r, dst[:max(r, 0)].tobytes()


def encode_hc(data, cap=None, impl: str = "port"):
    r, dst = _encode(data, cap, True, impl)
    return r, dst[:max(r, 0)].tobytes()


def decode_known(comp, osize: int, impl: str = "port"):
    """LZ4_uncompress semantics: returns (bytes_read or <0, output)."""
    src = _as_u8(comp)
    dst = np.zeros(max(osize, 0) + 64, dtype=np.uint8)
    if impl == "port":
        srcp = np.concatenate([src, np.zeros(16, np.uint8)])
        r = port().lz4o_decode_known(_u8p(srcp), src.size, _u8p(dst), osize)
    else:
        # the reference may read up to compressBound(osize) bytes: give it zero padding, never garbage
        srcp = np.concatenate([src, np.zeros(bound(max(osize, 0)) + 64, np.uint8)])
        r = ref().LZ4_uncompress(srcp.ctypes.data, dst.ctypes.data, osize)
    return int(r), dst[:max(osize, 0)].tobytes()


def decode_unknown(comp, max_out: int, impl: str = "port"):
    """LZ4_uncompress_unknownOutputSize semantics: returns (bytes_written or <0, output[:ret])."""
    src = _as_u8(comp)
    dst = np.zeros(max(max_out, 0) + 64, dtype=np.uint8)
    srcp = np.concatenate([src, np.zeros(16, np.uint8)])
    if impl == "port":
        r = port().lz4o_decode_unknown(_u8p(srcp), src.size, _u8p(dst), max_out)
    else:
        r = ref().LZ4_uncompress_unknownOutputSize(srcp.ctypes.data, dst.ctypes.data, src.size, max_out)
    return int(r), dst[:max(r, 0)].tobytes()


def mt_run(kind: str, impl: str, src: np.ndarray, src_off, src_len, dst: np.ndarray, dst_off, dst_cap, nthreads: int):
    """Run one CPU codec over a batch on `nthreads` host threads (CPU-baseline timing only).

    kind: 'encode' | 'encode_hc' | 'decode'.  Returns (seconds, out int32[n]).
    """
    p = port()
    if impl == "ref":
        lib = ref()
        fn = {"encode": lib.LZ4_compress_limitedOutput, "encode_hc": lib.LZ4_compressHC_limitedOutput,
              "decode": lib.LZ4_uncompress}[kind]
    else:
        fn = {"encode": p.lz4o_encode4, "encode_hc": p.lz4o_encode_hc4, "decode": p.lz4o_decode3}[kind]
    fnp = C.cast(fn, C.c_void_p)
    src_off = np.ascontiguousarray(src_off, dtype=np.int64)
    dst_off = np.ascontiguousarray(dst_off, dtype=np.int64)
    src_len = np.ascontiguousarray(src_len, dtype=np.int32)
    dst_cap = np.ascontiguousarray(dst_cap, dtype=np.int32)
    out = np.zeros(src_off.size, dtype=np.int32)
    secs = p.lz4o_mt_run(0 if kind != "decode" else 1, fnp, src.ctypes.data, src_off.ctypes.data, src_len.ctypes.data,
                         dst.ctypes.data, dst_off.ctypes.data, dst_cap.ctypes.data, out.ctypes.data,
                         int(src_off.size), int(nthreads))
    return float(secs), out
