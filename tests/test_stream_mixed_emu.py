"""The LZ4Stream frame steps of lz4_stream.cuh on the CPU warp emulator.

lz4b200_stream_encode_from_device writes each chunk's frame on the device (header bytes, then the payload from the
encoder's slot or, for a stored chunk, from the caller's source); lz4b200_stream_decode_to_device copies each stored
chunk's payload to its place in the output.  Here both steps run on the emulator: the frames must equal the reference
framing (the oracle stand-in's rules: LZ4Stream.cs:239-269, the HC bit on stored chunks too) at every varint length
boundary and every encoder result class, and both copies must be exact at every alignment without touching a byte around
them."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import emu
from tests.test_stream_host_logic import _varint

_P, _I, _U64 = C.c_void_p, C.c_int, C.c_uint64
_SIGNATURES = {                                                   # name: (restype, argtypes)
    "emu_stream_frame": (None, [_I, _P, _P, _P, _P, _P, _P, _P, _P, _U64]),
    "emu_stream_header": (_I, [_I, _I, _I, _P]),
    "emu_stream_stored": (None, [_I, _P, _P, _P, _U64]),
}
_slib = None


def _stream_lib():
    """The frame steps' harness unit (tests/simt_emu/emu_stream.cpp), built by the emulator driver's builder."""
    global _slib
    if _slib is None:
        l = C.CDLL(emu.build(os.path.join(os.path.dirname(os.path.abspath(emu.__file__)), "simt_emu", "emu_stream.cpp")))
        for name, (restype, argtypes) in _SIGNATURES.items():
            getattr(l, name).restype = restype
            getattr(l, name).argtypes = argtypes
        _slib = l
    return _slib


def _ptrs(addrs):
    return (C.c_void_p * len(addrs))(*addrs)


def _i32(v):
    return np.array(v, np.int32)


def _header(raw, r, hc):
    """The reference chunk header for a chunk of `raw` bytes whose encoder result (capacity = raw) is r."""
    comp = 0 < r < raw
    return _varint((1 if comp else 0) | (2 if hc else 0)) + _varint(raw) + (_varint(r) if comp else b"")


def _frame(data, r, comp, hc):
    return _header(len(data), r, hc) + (comp[:r] if 0 < r < len(data) else data)


def _red(n, skew, fill=0xCD):
    """A buffer with `n` usable bytes `skew` bytes past a 16-byte boundary, 48 red-zone bytes around them."""
    a = np.full(n + skew + 96, fill, np.uint8)
    lo = (-a.ctypes.data) % 16 + 32 + skew
    return a, lo


BOUNDARIES = [127, 128, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 28) - 1, 1 << 28]


def _results(raw):
    """Encoder results around every class: failed (<= 0), compressed at every varint boundary below raw, raw - 1 (the
    largest compressed), raw (did not shrink) and above raw."""
    rs = {-3, 0, 1, raw - 1, raw, raw + 1} | {b for b in BOUNDARIES if b < raw}
    return sorted(r for r in rs if r >= -3)


def test_headers_at_every_varint_boundary():
    """Header bytes (flags, varint(raw), varint(compLen)) of the frame step for raw and compLen on both sides of every
    varint length boundary, up to the largest raw length a frame may have (INT32_MAX - 11)."""
    out = np.zeros(16, np.uint8)
    raws = sorted({0, 1, 2, 126} | set(BOUNDARIES) | {b + 1 for b in BOUNDARIES} | {2 ** 31 - 12})
    n = 0
    for raw in raws:
        for r in _results(raw):
            for hc in (0, 1):
                h = _stream_lib().emu_stream_header(raw, r, hc, out.ctypes.data)
                assert out[:h].tobytes() == _header(raw, r, hc), (raw, r, hc)
                n += 1
    assert n > 250


def _run_frames(chunks, ss, ds, cs, seed):
    """chunks: (raw bytes, r, compressed bytes, hc).  Each chunk's source `ss`, compressed bytes `cs` and frame `ds` bytes
    past a 16-byte boundary, red zones around each.  Asserts the frames, their sizes and the red zones."""
    srcs, comps, dsts, keep = [], [], [], []
    for data, r, comp, hc in chunks:
        a, alo = _red(len(data), ss, 0x11)
        a[alo:alo + len(data)] = np.frombuffer(data, np.uint8)
        b, blo = _red(len(comp), cs, 0x22)
        b[blo:blo + len(comp)] = np.frombuffer(comp, np.uint8)
        want = _frame(data, r, comp, hc)
        f, flo = _red(len(want), ds)
        keep.append((a, b, f, flo, want))
        srcs.append(a.ctypes.data + alo); comps.append(b.ctypes.data + blo); dsts.append(f.ctypes.data + flo)
    n = len(chunks)
    out, size = np.zeros(n, np.int32), np.zeros(n, np.int32)
    raw, rr, hc = _i32([len(c[0]) for c in chunks]), _i32([c[1] for c in chunks]), _i32([int(c[3]) for c in chunks])
    _stream_lib().emu_stream_frame(n, _ptrs(srcs), raw.ctypes.data, _ptrs(comps), rr.ctypes.data, hc.ctypes.data,
                                   _ptrs(dsts), out.ctypes.data, size.ctypes.data, seed)
    for (data, r, _, h), (_, _, f, flo, want), o, s in zip(chunks, keep, out, size):
        who = (len(data), r, h, ss, ds, cs)
        assert o == s == len(want), who
        assert f[flo:flo + len(want)].tobytes() == want, who
        assert (f[:flo] == 0xCD).all() and (f[flo + len(want):] == 0xCD).all(), who


def _chunk(rng, raw, r, hc):
    data = rng.integers(0, 256, raw, dtype=np.uint8).tobytes()
    comp = rng.integers(0, 256, max(r, 0), dtype=np.uint8).tobytes() if 0 < r < raw else b""
    return data, r, comp, hc


def test_frames_at_every_varint_boundary_and_result_class():
    """Whole frames for raw on both sides of 127/128, 16383/16384 and 2^21 and every result class of each: failed,
    compressed at each varint boundary below raw, raw - 1, raw and above raw; fast and HC flags."""
    rng = np.random.default_rng(3)
    raws = [1, 2, 127, 128, 129, 16383, 16384, 16385, (1 << 21) - 1, 1 << 21, (1 << 21) + 1]
    chunks = [_chunk(rng, raw, r, hc) for raw in raws for r in _results(raw) for hc in (False, True)
              if raw < 16384 or r in (-3, raw - 1, raw, 128, 16384, (1 << 21) - 1)]
    _run_frames(chunks, 3, 5, 7, seed=11)
    _run_frames([_chunk(rng, 0, r, hc) for r in (-1, 0, 1) for hc in (False, True)], 0, 0, 0, seed=12)   # an empty chunk


LENGTHS = list(range(1, 181)) + [4096 + 7]


@pytest.mark.parametrize("ss", range(16))
def test_frame_copies_at_every_alignment(ss):
    """Stored frames (payload = the source) and compressed ones (payload = the encoder's bytes) at every source, slot and
    frame alignment mod 16, guard bytes around every frame."""
    rng = np.random.default_rng(ss)
    for ds in range(16):
        chunks = []
        for k, L in enumerate(LENGTHS if ds in (0, 9) else LENGTHS[::7]):
            r = L if k % 2 else max(L - 1 - k % 5, 0)               # stored (r == L, or r <= 0 for tiny L) / compressed
            chunks.append(_chunk(rng, L, r, bool(k % 3 == 0)))
        _run_frames(chunks, ss, ds, (ss + ds) % 16, seed=ss * 16 + ds)


def _run_stored(lens, stored_mask, ss, ds, seed):
    rng = np.random.default_rng(seed)
    srcs, dsts, keep = [], [], []
    for L in lens:
        a, alo = _red(L, ss, 0x11)
        a[alo:alo + L] = rng.integers(0, 256, L, dtype=np.uint8)
        b, blo = _red(L, ds)
        keep.append((a, alo, b, blo))
        srcs.append(a.ctypes.data + alo); dsts.append(b.ctypes.data + blo)
    st = _i32([L if s else 0 for L, s in zip(lens, stored_mask)])
    _stream_lib().emu_stream_stored(len(lens), _ptrs(srcs), st.ctypes.data, _ptrs(dsts), seed)
    for L, s, (a, alo, b, blo) in zip(lens, stored_mask, keep):
        who = (L, s, ss, ds)
        if s:
            assert (b[blo:blo + L] == a[alo:alo + L]).all(), who
            assert (b[:blo] == 0xCD).all() and (b[blo + L:] == 0xCD).all(), who
        else:
            assert (b == 0xCD).all(), who                          # a compressed chunk: the step writes nothing


@pytest.mark.parametrize("ss", range(16))
def test_stored_copy_at_every_alignment(ss):
    """The decode's stored copy at every source and destination alignment mod 16, lengths 0-300 and two large ones, red
    zones around every output; compressed chunks in the same batch are left alone."""
    lens = list(range(0, 301)) + [4096 + 7, 65536 + 3]
    for ds in range(16):
        ls = lens if ds in (0, 7) else lens[:301:3]
        _run_stored(ls, [k % 4 != 1 for k in range(len(ls))], ss, ds, seed=ss * 16 + ds)


def test_stored_copy_across_varint_boundaries():
    lens = [127, 128, 16383, 16384, (1 << 21) - 1, 1 << 21, (1 << 21) + 1]
    _run_stored(lens, [True] * len(lens), 5, 11, seed=3)
