"""The device header walk of the LZ4Stream decode from a size the device wrote (lz4_stream.cuh stream_walk_stage) on the
CPU warp emulator, against the host walk it restates (framing.cpp stream_walk, compiled into the same harness).

lz4b200_stream_decode_to_device_at_async reads the stream's size S on the device, so the headers cannot be walked on the
host.  The host cuts K = ceil(dst_cap / block_size) chunk slots into stages of `per`; one warp per stage walks the headers
from the carry cells the previous stage left and writes the stage's FRAMED_DECODE entries and its span.  Here every stage
runs on the emulator over constructed streams, and the result, the entries and the spans are checked against a
restatement built on the host walk's chunks: the first malformed header is E_FORMAT, the first chunk that breaks a bound
(rawLen > block_size, a (K+1)-th chunk, output past dst_cap) E_ARG, S outside [0, src_cap] E_ARG before any read.  A
separate process fences the source with PROT_NONE pages, so a read outside the aligned 16-byte units around [src, src + S)
fails the test instead of the session."""
import ctypes as C
import hashlib
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from tests import emu

_P, _I, _L, _U64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
E_ARG, E_FORMAT = -1, -5
HEADER_MAX = 30
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_wlib = None


def _lib():
    """The walk's harness unit (tests/simt_emu/emu_stream_walk.cpp); keyed on framing.cpp too, which it compiles in."""
    global _wlib
    if _wlib is None:
        with open(os.path.join(ROOT, "lz4net_b200", "csrc", "framing.cpp"), "rb") as f:
            key = hashlib.sha256(f.read()).hexdigest()[:16]
        l = C.CDLL(emu.build(os.path.join(ROOT, "tests", "simt_emu", "emu_stream_walk.cpp"), (f"-DFRAMING_SHA={key}",)))
        l.emu_stream_walk.restype = _L
        l.emu_stream_walk.argtypes = [_P, _L, _P, _I, _L, _I, _I, _I, _L, _P, _P, _P, _P, _P, _P, _U64]
        l.emu_stream_walk_result.restype = _L
        l.emu_stream_walk_result.argtypes = [_P, C.c_int]
        l.emu_host_walk.restype = _L
        l.emu_host_walk.argtypes = [_P, _L, _P, _P, _P, _P, _L, _P]
        l.emu_stream_walk_header_max.restype = _I
        _wlib = l
    return _wlib


# ---- constructing streams -------------------------------------------------------------------------------------------
def varint(v, pad=0):
    """LZ4Stream's varint of v, padded with `pad` extra continuation bytes (a longer encoding the reader accepts)."""
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            break
    if pad:
        out[-1] |= 0x80
        out += b"\x80" * (pad - 1) + b"\x00"
    return bytes(out)


def chunk(raw, payload=None, comp=None, flags=None, pads=(0, 0, 0)):
    """One chunk: stored (payload = raw bytes) or compressed (comp = its payload bytes)."""
    if comp is None:
        body = payload if payload is not None else (np.arange(raw) % 251).astype(np.uint8).tobytes()
        f = 0 if flags is None else flags
        return varint(f, pads[0]) + varint(raw, pads[1]) + body
    f = 1 if flags is None else flags
    return varint(f, pads[0]) + varint(raw, pads[1]) + varint(len(comp), pads[2]) + comp


def _aligned(nbytes, align):
    raw = np.zeros(nbytes + 48, np.uint8)
    start = (-raw.ctypes.data) % 16 + align
    return raw[start:start + nbytes]


# ---- the restatement ------------------------------------------------------------------------------------------------
def host_walk(stream):
    """framing.cpp stream_walk: (total or E_FORMAT, [(payload, raw, stored bytes, compressed)] before it returned)."""
    n = len(stream)
    buf = np.frombuffer(stream, np.uint8) if n else np.zeros(1, np.uint8)
    cap = n + 1
    pay, raw, ln = np.zeros(cap, np.int64), np.zeros(cap, np.int32), np.zeros(cap, np.int32)
    comp, count = np.zeros(cap, np.uint8), C.c_int64()
    r = _lib().emu_host_walk(buf.ctypes.data, n, pay.ctypes.data, raw.ctypes.data, ln.ctypes.data, comp.ctypes.data, cap,
                             C.byref(count))
    k = count.value
    return r, list(zip(pay[:k].tolist(), raw[:k].tolist(), ln[:k].tolist(), comp[:k].astype(bool).tolist()))


def expected(stream, src_cap, S, block_size, dst_cap):
    """The call's result and the chunks the walk accepts, by the contract."""
    if S < 0 or S > src_cap:
        return E_ARG, []
    K = -(-dst_cap // block_size)
    r, chunks = host_walk(stream[:S])
    total, ok = 0, []
    for j, (pay, raw, ln, comp) in enumerate(chunks):
        if j >= K or raw > block_size or total + raw > dst_cap:
            return E_ARG, ok
        ok.append((pay, raw, ln, comp, total))
        total += raw
    return r, ok


def plan(dst_cap, block_size, per):
    K = -(-dst_cap // block_size)
    stages = max(1, -(-K // per))
    return K, stages, K - (stages - 1) * per


def walk(src, src_cap, S, block_size, dst_cap, per, seed=1, size_cell=None):
    """Runs every stage; returns (result, entries (so, dof, sl, dc, stored) per slot, lift descriptors per stage)."""
    K, stages, m_last = plan(dst_cap, block_size, per)
    slots = max(K, 1)
    so, dof = np.full(slots, -7, np.int64), np.full(slots, -7, np.int64)
    sl, dc, st = np.full(slots, -7, np.int32), np.full(slots, -7, np.int32), np.full(slots, -7, np.int32)
    lift = np.zeros(8 * stages, np.int64)
    cell = np.array([S], np.int64) if size_cell is None else size_cell
    r = _lib().emu_stream_walk(src, src_cap, cell.ctypes.data, block_size, dst_cap, per, stages, m_last,
                               per * (block_size + HEADER_MAX), so.ctypes.data, dof.ctypes.data, sl.ctypes.data, dc.ctypes.data,
                               st.ctypes.data, lift.ctypes.data, seed)
    return r, list(zip(so[:K].tolist(), dof[:K].tolist(), sl[:K].tolist(), dc[:K].tolist(), st[:K].tolist())), lift.reshape(stages, 8)


def check(stream, block_size, dst_cap, per, align=0, S=None, src_cap=None, seed=1):
    """Walks `stream` at host alignment `align` and checks result, entries and spans.  Returns the result."""
    S = len(stream) if S is None else S
    src_cap = len(stream) if src_cap is None else src_cap
    src = _aligned(max(len(stream), 1), align)
    src[:len(stream)] = np.frombuffer(stream, np.uint8)
    addr = src.ctypes.data
    want, ok = expected(stream, src_cap, S, block_size, dst_cap)
    r, entries, lift = walk(addr, src_cap, S, block_size, dst_cap, per, seed)
    assert r == want, (r, want)
    # the spans: stage k covers the frames of its accepted chunks, back to back from where stage k-1 ended
    spans, cur = [], 0
    for k in range(len(lift)):
        mine = [c for j, c in enumerate(ok) if j // per == k]
        end = mine[-1][0] + mine[-1][2] if mine else cur
        spans.append((cur, end))
        cur = end
    for k, (lo, hi) in enumerate(spans):
        slot0, slot1, s0, s1, s2 = lift[k][:5].tolist()
        bound = int(lift[k][5:6].view(np.int32)[0])
        assert (slot0, s0, s1, s2) == (0, lo, hi, hi), (k, lift[k][:5], lo, hi)
        assert slot1 == (hi - lo + 32 + 15) // 16 * 16 and bound == per * (block_size + HEADER_MAX)
    for j, e in enumerate(entries):
        if j < len(ok) and ok[j][1] > 0:
            pay, raw, ln, comp, at = ok[j]
            lo = spans[j // per][0]
            so = (addr + lo) % 16 + pay - lo
            assert e == ((so, at, ln, raw, 0) if comp else (so, at, 0, 0, raw)), (j, e, ok[j])
        else:
            assert e == (0, 0, 0, 0, -1), (j, e)                          # neutral: empty, past the end, after a status
    return r


# ---- well-formed streams --------------------------------------------------------------------------------------------
def _mixed(rng, n, block_size, empty=True):
    out = b""
    for _ in range(n):
        raw = int(rng.integers(0 if empty else 1, block_size + 1))
        kind = int(rng.integers(0, 4))
        if kind == 0:
            out += chunk(raw, flags=2)                                     # stored, HC-flagged
        elif kind == 1 and raw > 0:
            out += chunk(raw, comp=bytes(rng.integers(0, 256, int(rng.integers(0, raw + 1)), dtype=np.uint8)), flags=3)
        elif kind == 2 and raw > 0:
            out += chunk(raw, comp=bytes(raw))                             # compLen == rawLen, compressed flag
        else:
            out += chunk(raw)
    return out


@pytest.mark.parametrize("per", [1, 2, 3, 7])
@pytest.mark.parametrize("align", [0, 1, 9, 15])
def test_well_formed_streams_match_the_host_walk(per, align):
    rng = np.random.default_rng(100 * per + align)
    for bs in (1, 16, 200, 5000):
        n = int(rng.integers(1, 12))
        s = _mixed(rng, n, bs)
        total = host_walk(s)[0]
        assert total >= 0
        for dst_cap in (total, n * bs, n * bs + 3 * bs):
            if dst_cap >= total and -(-dst_cap // bs) >= n:
                assert check(s, bs, dst_cap, per, align, seed=per + align) == total


@pytest.mark.parametrize("nbytes", [1, 2, 3, 4, 5])
def test_varints_of_one_to_five_bytes(nbytes):
    v = [5, 200, 20000, 3_000_000, 300_000_000][nbytes - 1]
    assert len(varint(v)) == nbytes
    # rawLen of nbytes bytes (a compressed chunk's payload is short whatever its rawLen), then a stored one
    s = chunk(v, comp=bytes(range(4))) + chunk(3)
    assert check(s, v, v + 3, 2) == v + 3
    if v < (1 << 16):
        assert check(chunk(v) + chunk(v, comp=bytes(min(v, 9))), v, 2 * v, 1) == 2 * v
    # compLen of nbytes bytes: a longer encoding of a small value
    s = chunk(40, comp=bytes(range(30)), pads=(0, 0, nbytes - 1)) + chunk(7)
    assert check(s, 40, 47, 1) == 47


@pytest.mark.parametrize("pads", [(1, 2, 3), (4, 4, 4), (9, 0, 0), (0, 9, 9), (9, 9, 9)])
def test_headers_up_to_thirty_bytes(pads):
    s = chunk(40, comp=bytes(range(30)), pads=pads) + chunk(7, pads=pads[:2] + (0,)) + chunk(1, pads=pads)
    assert host_walk(s)[0] == 48
    for per in (1, 2, 3):
        assert check(s, 40, 120, per, align=per * 5) == 48


def test_empty_chunks_count_as_chunks_and_get_the_neutral_entry():
    s = chunk(0) + chunk(5) + chunk(0, comp=b"") + chunk(0, flags=2) + chunk(3)
    assert check(s, 8, 40, 2) == 8                                         # K = 5: every chunk has its slot
    assert check(s, 8, 16, 1) == E_ARG                                     # K = 2: the third chunk is one too many
    assert check(chunk(0) * 3, 4, 12, 3) == 0


def test_streams_that_end_early_pad_the_rest():
    s = chunk(10) + chunk(10, comp=bytes(4))
    for per in (1, 2, 3):
        assert check(s, 10, 100, per) == 20                                # K = 10 slots, two chunks
    assert check(b"", 10, 100, 4) == 0
    assert check(b"", 10, 0, 4) == 0                                       # no slots at all


# ---- malformed streams ----------------------------------------------------------------------------------------------
MALFORMED = {
    "truncated flags varint": chunk(4) + b"\x81",
    "truncated raw varint": chunk(4) + b"\x00\x85",
    "truncated compLen varint": chunk(4) + b"\x01\x05\x83",
    "header without rawLen": chunk(4) + b"\x00",
    "ten-byte varint then a short read": b"\x80" * 9 + b"\x80" + b"\x05" + b"ab",
    "rawLen casts negative": b"\x00" + varint(1 << 31) + b"x",
    "rawLen casts negative, ten bytes": b"\x00" + b"\xff" * 9 + b"\x01" + b"x",
    "compLen casts negative": b"\x01\x05" + varint((1 << 32) - 3) + b"abc",
    "compLen above rawLen": b"\x01\x03\x04abcd",
    "payload past S": chunk(4) + b"\x00\x09abc",
    "compressed payload past S": b"\x01\x09\x05abcd",
    "compressed with flags >> 2": b"\x05\x04\x02ab",
    "compressed with a high flag bit": varint(1 | (1 << 40)) + b"\x04\x02ab",
}


@pytest.mark.parametrize("name", sorted(MALFORMED))
@pytest.mark.parametrize("per", [1, 2, 3])
def test_malformed_streams(name, per):
    s = MALFORMED[name]
    r = check(s, 1 << 20, 1 << 22, per)
    assert r == host_walk(s)[0]
    assert r == E_FORMAT or name.startswith("ten-byte")


def test_a_ten_byte_varint_is_read_as_the_host_reads_it():
    # the count >= 64 exit: ten continuation bytes end the varint; the value keeps its low 64 bits
    s = b"\x80" * 9 + b"\x00" + b"\x05" + b"hello"
    assert host_walk(s)[0] == 5 and check(s, 8, 5, 1) == 5
    s = b"\x80" * 10 + b"\x05" + b"hello"                                  # the tenth byte still has its continuation bit
    assert check(s, 8, 5, 1) == host_walk(s)[0] == 5


def test_a_stored_chunk_with_high_flags_is_accepted():
    s = chunk(6, flags=4) + chunk(6, flags=0xFE)
    assert check(s, 8, 12, 1) == 12 == host_walk(s)[0]


def test_the_first_event_wins():
    bad = MALFORMED["compLen above rawLen"]
    # a bound broken before the malformed header: E_ARG; after it: E_FORMAT
    assert check(chunk(20) + bad, 10, 100, 2) == E_ARG
    assert check(chunk(5) + bad + chunk(20), 10, 100, 2) == E_FORMAT
    assert check(chunk(5) * 3 + bad, 5, 15, 2) == E_FORMAT              # the (K+1)-th header is malformed: E_FORMAT
    assert check(chunk(5) * 4, 5, 15, 2) == E_ARG                         # a well-formed (K+1)-th chunk: E_ARG


# ---- the three bounds, and the size check ---------------------------------------------------------------------------
@pytest.mark.parametrize("per", [1, 2, 3])
def test_the_three_bounds(per):
    s = chunk(8) + chunk(8, comp=bytes(3)) + chunk(8)
    assert check(s, 8, 24, per) == 24
    assert check(s, 7, 24, per) == E_ARG                                   # rawLen > block_size
    assert check(s, 8, 23, per) == E_ARG                                   # output past dst_cap (K = 3 still)
    assert check(s, 8, 16, per) == E_ARG                                   # K = 2: a third chunk
    assert check(s, 12, 24, per) == E_ARG                                  # K = 2 at block_size 12, though 24 bytes fit
    assert check(chunk(4) * 6, 8, 24, per) == E_ARG                        # six chunks, K = 3


def test_size_out_of_range_reads_nothing():
    s = chunk(8) + chunk(8)
    for S, cap in ((-1, len(s)), (len(s) + 1, len(s)), (5, 4), (1, 0)):
        assert check(s, 8, 16, 2, S=S, src_cap=cap) == E_ARG
    # the source is never touched: a null source with S out of range, and an empty one
    r, entries, _ = walk(None, 0, 3, 8, 16, 2)
    assert r == E_ARG and all(e == (0, 0, 0, 0, -1) for e in entries)
    assert walk(None, 0, 0, 8, 16, 2)[0] == 0


def test_a_prefix_of_the_source():
    s = chunk(8) + chunk(8) + b"\xff\xff"
    assert check(s, 8, 16, 1, S=len(s) - 2) == 16
    assert check(s, 8, 16, 1, S=len(s) - 1) == E_FORMAT                   # the stray byte is a truncated header


def test_result_priority():
    res = lambda cells, failed: _lib().emu_stream_walk_result(np.array(cells, np.int64).ctypes.data, failed)  # noqa: E731
    assert res([10, 99, E_ARG, 10], 1) == E_ARG                             # the walk's status first
    assert res([10, 99, E_FORMAT, 10], 0) == E_FORMAT
    assert res([7, 99, 0, 10], 1) == E_ARG                                  # then a cursor short of S
    assert res([10, 99, 0, 10], 1) == E_FORMAT                              # then a chunk that did not decode
    assert res([10, 99, 0, 10], 0) == 99


def test_the_header_bound_is_the_host_walks():
    assert _lib().emu_stream_walk_header_max() == HEADER_MAX == 3 * 10


def test_random_streams_and_stage_plans():
    rng = np.random.default_rng(7)
    for trial in range(40):
        bs = int(rng.choice([1, 3, 16, 100, 700]))
        s = _mixed(rng, int(rng.integers(0, 30)), bs)
        if trial % 3 == 0 and s:
            cut = int(rng.integers(0, len(s)))                              # damage: truncate, or flip a byte
            s = s[:cut] if trial % 2 else s[:cut] + bytes([s[cut] ^ 0x81]) + s[cut + 1:]
        total = max(0, host_walk(s)[0])
        dst_cap = max(0, total + int(rng.integers(-bs, 3 * bs)))
        check(s, bs, dst_cap, int(rng.integers(1, 6)), int(rng.integers(0, 16)), seed=trial)


# ---- nothing outside the aligned units around [src, src + S) is read -------------------------------------------------
_FENCED = textwrap.dedent("""
    import ctypes as C, mmap, sys
    import numpy as np
    from tests import test_stream_walk_emu as t
    a, b = int(sys.argv[1]), int(sys.argv[2])
    page = mmap.PAGESIZE
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    m = mmap.mmap(-1, 4 * page)
    base = C.addressof(C.c_char.from_buffer(m))
    # pages 0 and 3 are PROT_NONE; the stream starts a bytes into page 1 and ends b bytes before page 3
    S = 2 * page - a - b
    rng = np.random.default_rng(a * 16 + b)
    body = t.chunk(1000, comp=bytes(rng.integers(0, 256, 700, dtype=np.uint8))) + t.chunk(0) + t.chunk(3)
    body += t.chunk(300, pads=(3, 3, 0))
    tail = S - len(body)
    hdr = next(h for h in (t.varint(0) + t.varint(tail - k) for k in range(2, 7)) if len(h) + (tail - len(h)) == tail and
               h == t.varint(0) + t.varint(tail - len(h)))                          # a stored chunk that ends exactly at S
    stream = body + hdr + bytes(rng.integers(0, 256, S - len(body) - len(hdr), dtype=np.uint8))
    assert len(stream) == S
    m[page + a:page + a + S] = stream
    assert libc.mprotect(base, page, 0) == 0 and libc.mprotect(base + 3 * page, page, 0) == 0
    src = base + page + a
    for per, dst_cap in ((1, 5 * 8192), (3, 6 * 8192), (8, 8 * 8192)):
        want = t.expected(stream, S, S, 8192, dst_cap)[0]
        r = t.walk(src, S, S, 8192, dst_cap, per)[0]
        assert r == want and r > 0, (r, want)
    # a stream cut short: its last header is read up to the size given and no further
    for cut in (1, 2, 5):
        r = t.walk(src, S, len(body) + cut, 8192, 8 * 8192, 2)[0]
        assert r == t.expected(stream, S, len(body) + cut, 8192, 8 * 8192)[0] == -5
    print("ok")
""")


@pytest.mark.parametrize("a,b", [(0, 0), (1, 0), (0, 1), (15, 15), (7, 9), (3, 14)])
def test_nothing_outside_the_aligned_units_around_the_stream_is_read(a, b):
    _lib()                                                                 # build here, so the child only loads it
    r = subprocess.run([sys.executable, "-c", _FENCED, str(a), str(b)], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
