"""The Wrap / Unwrap packet steps of lz4_wrap.cuh on the CPU warp emulator.

The device calls lz4b200_wrap_batch_device / unwrap_batch_device / unwrap_batch_packed run the existing codec between a
prep and a finish step per packet.  Here the steps themselves run on the emulator: the header rules must agree with the
host framing (lz4b200_unwrap_size), the stored copies must be exact at every alignment without touching a byte around
them, and the neutral decode entry given to stored and rejected packets must make every decoder read and write nothing."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

from tests import emu

E_ARG, E_FORMAT = -1, -5

_P, _I, _U64 = C.c_void_p, C.c_int, C.c_uint64
_SIGNATURES = {                                                   # name: (restype, argtypes)
    "emu_unwrap_prep": (None, [_I, _P, _P, _P, _P, _P, _P, _U64]),
    "emu_wrap_finish": (None, [_I, _P, _P, _P, _P, _P, _P, _U64]),
    "emu_unwrap_finish": (None, [_I, _P, _P, _P, _P, _P, _P, _P, _U64]),
}
_wlib = None


def _wrap_lib():
    """The packet steps' harness unit (tests/simt_emu/emu_wrap.cpp), built by the emulator driver's builder."""
    global _wlib
    if _wlib is None:
        l = C.CDLL(emu.build(os.path.join(os.path.dirname(os.path.abspath(emu.__file__)), "simt_emu", "emu_wrap.cpp")))
        for name, (restype, argtypes) in _SIGNATURES.items():
            getattr(l, name).restype = restype
            getattr(l, name).argtypes = argtypes
        _wlib = l
    return _wlib


def _host():
    from lz4net_b200 import build, native
    build.build()
    return native.lib()


def _ptrs(addrs):
    return (C.c_void_p * len(addrs))(*addrs)


def _i32(v):
    return np.array(v, np.int32)


def _unwrap_prep(packets, caps=None, fence=None, seed=1):
    """The prep step over `packets` (bytes); returns (sizes, dec_len, dec_cap)."""
    n = len(packets)
    size, dl, dc = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
    lens = _i32([len(p) for p in packets])
    cps = None if caps is None else _i32(caps)
    with emu._staged(packets, 0, fence) as src:
        _wrap_lib().emu_unwrap_prep(n, _ptrs(src), lens.ctypes.data, None if cps is None else cps.ctypes.data,
                                    size.ctypes.data, dl.ctypes.data, dc.ctypes.data, seed)
    return size.tolist(), dl.tolist(), dc.tolist()


def _header_cases():
    rng = np.random.default_rng(31)
    out = []
    for n in range(17):
        for k in range(60):
            b = bytearray(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
            if n >= 8:
                raw, stored = [(int(rng.integers(0, 40)), int(rng.integers(0, n - 7))),      # valid stored / compressed
                               (int(rng.integers(0, 40)), n - 8),                            # stored field at the limit
                               (int(rng.integers(0, 40)), n - 7),                            # oversized by one
                               (int(rng.integers(0, 1 << 32)), int(rng.integers(0, 1 << 32))),  # random (negative fields)
                               (0x80000000 | int(rng.integers(0, 1 << 31)), 0),              # negative raw
                               (1, 0x80000000 | int(rng.integers(0, 1 << 31))),              # negative stored
                               (5, 5), (0, 0)][k % 8]
                if raw > n - 8 and k % 8 == 6:
                    raw = stored = n - 8
                b[:8] = struct.pack("<II", raw, stored)
            out.append(bytes(b))
    return out


def test_header_rules_match_the_host_framing():
    host = _host()
    packets = _header_cases()
    want = []
    for p in packets:
        buf = C.create_string_buffer(p, max(len(p), 1))
        want.append(host.lz4b200_unwrap_size(buf, len(p)))
    size, dl, dc = _unwrap_prep(packets, seed=5)
    assert size == want
    assert any(w == E_FORMAT for w in want) and sum(w >= 0 for w in want) > 100
    for p, s, l, c in zip(packets, size, dl, dc):
        if s >= 0:
            raw, stored = struct.unpack("<ii", p[:8])
            assert (l, c) == ((stored, raw) if stored < raw else (0, 0))             # compressed: a decode entry
        else:
            assert (l, c) == (0, 0)                                                  # rejected: neutral
    # a capacity: one byte short of the size is LZ4B200_E_ARG (framing.cpp:243), the size itself passes
    ok = [i for i, s in enumerate(size) if s >= 0]
    exact, _, _ = _unwrap_prep([packets[i] for i in ok], [size[i] for i in ok], seed=6)
    short, sdl, sdc = _unwrap_prep([packets[i] for i in ok], [size[i] - 1 for i in ok], seed=7)
    assert exact == [size[i] for i in ok]
    assert short == [E_ARG] * len(ok) and set(sdl) == {0} and set(sdc) == {0}


@pytest.mark.parametrize("fence", ["behind", "front"])
def test_header_reads_stay_inside_the_packet(fence):
    """Packets of 0-16 bytes against a PROT_NONE page: a read of any byte outside the packet would fault."""
    host = _host()
    for p in _header_cases()[::7]:
        buf = C.create_string_buffer(p, max(len(p), 1))
        assert _unwrap_prep([p], fence=fence)[0] == [host.lz4b200_unwrap_size(buf, len(p))]


def _red(n, skew, fill=0xCD):
    """A buffer with `n` usable bytes `skew` bytes past a 16-byte boundary, 48 red-zone bytes around them."""
    a = np.full(n + skew + 96, fill, np.uint8)
    base = a.ctypes.data
    lo = (-base) % 16 + 32 + skew
    return a, lo


LENGTHS = list(range(0, 301)) + [4096 + 7, 65536 + 3]


def _wrap_stored(lens, ss, ds, seed):
    """The wrap finish step with the encoder's result 0 (did not fit): every packet is stored.  Returns nothing; asserts."""
    rng = np.random.default_rng(seed)
    n = len(lens)
    ins, outs, src, dst = [], [], [], []
    for L in lens:
        a, lo = _red(L, ss, 0x11)
        a[lo:lo + L] = rng.integers(0, 256, L, dtype=np.uint8)
        b, blo = _red(L + 8, ds)
        ins.append((a, lo)); outs.append((b, blo))
        src.append(a.ctypes.data + lo); dst.append(b.ctypes.data + blo)
    res = np.zeros(n, np.int32)
    ln, cp, r0 = _i32(lens), _i32([L + 8 for L in lens]), _i32([0] * n)
    _wrap_lib().emu_wrap_finish(n, _ptrs(src), ln.ctypes.data, cp.ctypes.data, r0.ctypes.data, _ptrs(dst), res.ctypes.data, seed)
    for L, (a, lo), (b, blo), r in zip(lens, ins, outs, res):
        assert r == L + 8
        assert b[blo:blo + 8].tobytes() == struct.pack("<II", L, L)
        assert (b[blo + 8:blo + 8 + L] == a[lo:lo + L]).all(), (L, ss, ds)
        assert (b[:blo] == 0xCD).all() and (b[blo + 8 + L:] == 0xCD).all(), (L, ss, ds)


def _unwrap_stored(lens, ss, ds, seed):
    rng = np.random.default_rng(seed)
    n = len(lens)
    ins, outs, src, dst = [], [], [], []
    for L in lens:
        a, lo = _red(L + 8, ss, 0x11)
        a[lo:lo + 8] = np.frombuffer(struct.pack("<II", L, L), np.uint8)
        a[lo + 8:lo + 8 + L] = rng.integers(0, 256, L, dtype=np.uint8)
        b, blo = _red(L, ds)
        ins.append((a, lo)); outs.append((b, blo))
        src.append(a.ctypes.data + lo); dst.append(b.ctypes.data + blo)
    res = np.zeros(n, np.int32)
    z, ln, rd = _i32([0] * n), _i32(lens), _i32([-1] * n)
    _wrap_lib().emu_unwrap_finish(n, _ptrs(src), ln.ctypes.data, z.ctypes.data, z.ctypes.data, rd.ctypes.data,
                                  _ptrs(dst), res.ctypes.data, seed)
    for L, (a, lo), (b, blo), r in zip(lens, ins, outs, res):
        assert r == L
        assert (b[blo:blo + L] == a[lo + 8:lo + 8 + L]).all(), (L, ss, ds)
        assert (b[:blo] == 0xCD).all() and (b[blo + L:] == 0xCD).all(), (L, ss, ds)


@pytest.mark.parametrize("ss", range(16))
def test_wrap_stored_copy_at_every_alignment(ss):
    for ds in range(16):
        _wrap_stored(LENGTHS if ds in (0, 7) else LENGTHS[:301], ss, ds, seed=ss * 16 + ds)


@pytest.mark.parametrize("ss", range(16))
def test_unwrap_stored_copy_at_every_alignment(ss):
    for ds in range(16):
        _unwrap_stored(LENGTHS if ds in (0, 9) else LENGTHS[:301], ss, ds, seed=ss * 16 + ds)


def test_wrap_finish_header_and_statuses():
    """A compressed result writes the header only (the payload is the encoder's); invalid packets write nothing."""
    cases = [  # (len, cap, r) -> out_len
        (100, 108, 40, 48), (100, 108, 99, 107), (100, 108, 100, 108), (100, 108, 0, 108), (100, 108, -3, 108),
        (0, 8, 0, 8), (0, 8, 5, 8), (100, 107, 40, E_ARG), (-1, 100, 0, E_ARG), (0, 7, 0, E_ARG), (5, 1 << 30, 1, 9),
    ]
    n = len(cases)
    ins, outs, src, dst = [], [], [], []
    for L, cap, _, _ in cases:
        a, lo = _red(max(L, 0), 3, 0x11)
        b, blo = _red(max(cap, 0) if cap < 4096 else 64, 5)
        ins.append((a, lo)); outs.append((b, blo))
        src.append(a.ctypes.data + lo); dst.append(b.ctypes.data + blo)
    res = np.zeros(n, np.int32)
    ln, cp, r = (_i32([c[k] for c in cases]) for k in range(3))
    _wrap_lib().emu_wrap_finish(n, _ptrs(src), ln.ctypes.data, cp.ctypes.data, r.ctypes.data, _ptrs(dst), res.ctypes.data, 3)
    for (L, cap, r, want), (b, blo), got in zip(cases, outs, res):
        assert got == want, (L, cap, r)
        if want < 0:
            assert (b == 0xCD).all()
        else:
            stored = want - 8
            assert b[blo:blo + 8].tobytes() == struct.pack("<II", L, stored)
            if stored < L:
                assert (b[blo + 8:] == 0xCD).all()


def test_unwrap_finish_statuses():
    """Rejected packets keep their status and write nothing; a compressed packet restores raw bytes only when the decoder
    read exactly the stored bytes (framing.cpp:252)."""
    cases = [  # (size, dec_len, dec_cap, read) -> out_len
        (E_FORMAT, 0, 0, -1, E_FORMAT), (E_ARG, 0, 0, -1, E_ARG), (500, 40, 500, 40, 500), (500, 40, 500, 39, E_FORMAT),
        (500, 40, 500, -7, E_FORMAT), (1, 0, 1, -1, E_FORMAT), (0, 0, 0, -1, 0),
    ]
    n = len(cases)
    src, dst, bufs = [], [], []
    for _ in cases:
        a, lo = _red(64, 0, 0x11)
        b, blo = _red(64, 1)
        bufs.append((a, b)); src.append(a.ctypes.data + lo); dst.append(b.ctypes.data + blo)
    res = np.zeros(n, np.int32)
    size, dl, dc, rd = (_i32([c[k] for c in cases]) for k in range(4))
    _wrap_lib().emu_unwrap_finish(n, _ptrs(src), size.ctypes.data, dl.ctypes.data, dc.ctypes.data, rd.ctypes.data,
                                  _ptrs(dst), res.ctypes.data, 4)
    assert res.tolist() == [c[4] for c in cases]
    for _, b in bufs:
        assert (b == 0xCD).all()


@pytest.mark.parametrize("fence", ["behind", "front"])
@pytest.mark.parametrize("lanes", [4, 8, 16, 32, 104, 108, 116, 132, 1, 2])
def test_neutral_entries_read_and_write_nothing(lanes, fence):
    """The entry (src_len 0, dst_cap 0) that stored and rejected packets get: each decoder header the emulator runs (group
    kernels, output-staged group kernels, the lane-per-block decoder in both geometries) returns a negative result for it
    with its stream pointer against a PROT_NONE page and leaves every red-zone byte of its destination unchanged, in a
    batch mixed with real blocks."""
    import oracle
    from tests import cases
    d = cases.content("E50", 3000, seed=2).tobytes()
    c = oracle.encode(d)[1]
    k = 40
    with emu._fenced(b"", fence, 0) as empty:
        real = np.frombuffer(c, np.uint8).copy()
        src = [empty if i % 3 else real.ctypes.data for i in range(k)]
        isz = _i32([0 if i % 3 else len(c) for i in range(k)])
        caps = [0 if i % 3 else len(d) for i in range(k)]
        out = emu._Slots(caps, 5)
        res = np.full(k, 77, np.int32)
        cps = _i32(caps)
        args = (1, k, _ptrs(src), isz.ctypes.data, _ptrs(out.ptrs), cps.ctypes.data, res.ctypes.data, 9)    # known size
        if lanes in (1, 2):
            emu.lib().emu_decode_lpb(lanes - 1, *args)
        else:
            emu.lib().emu_decode(lanes, *args)
        got = out.take(caps, "decoder")
    for i in range(k):
        if i % 3:
            assert res[i] < 0 and got[i] == b""
        else:
            assert res[i] == len(c) and got[i] == d
