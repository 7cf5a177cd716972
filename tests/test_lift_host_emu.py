"""The staging step of the asynchronous decode and Unwrap from device-written offsets (lz4_lift.cuh) on the CPU warp
emulator.

lz4b200_decode_batch_to_device_at_async and lz4b200_unwrap_batch_to_device_at_async take the block offsets an
asynchronous offload wrote on the device, so the host cannot give a copy engine the range to stage.  The host cuts the
stages by each block's bound and gives every block a slot of the 16-aligned (bound + 32) bytes; on the device, one step
per stage validates each span, writes the decoder's entry, and gathers the spans' bytes into their slots by aligned
16-byte unit.  Here the step runs on the emulator over real host buffers against a NumPy restatement of the contract: a
well-formed span lands in its slot at the alignment mod 16 of its host address with exactly its bytes, a rejected one gets
the neutral entry (src_len 0, dst_cap 0), nothing of its slot is written and its result becomes LZ4B200_E_ARG.  A
separate process fences the source with PROT_NONE pages, so a read outside the aligned units around [src, src + src_cap)
fails the test instead of the session."""
import ctypes as C
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from tests import emu

_P, _I, _L, _U64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
_llib = None
E_ARG = -1
IO_FILL = 0xAB
DC = 777                                                                 # the caller's dst_cap, as the host uploads it
OUT = 5                                                                  # the decoder's result, before the status step
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    """The step's harness unit (tests/simt_emu/emu_lift.cpp), built by the emulator driver's builder."""
    global _llib
    if _llib is None:
        l = C.CDLL(emu.build(os.path.join(os.path.dirname(os.path.abspath(emu.__file__)), "simt_emu", "emu_lift.cpp")))
        l.emu_lift_stage.restype = None
        l.emu_lift_stage.argtypes = [_P, _L, _P, _P, _I, _P, _P, _P, _P, _P, _P, _U64]
        l.emu_lift_slot_bytes.restype = _L
        l.emu_lift_slot_bytes.argtypes = [_I]
        _llib = l
    return _llib


def _aligned(nbytes, align, fill):
    """A uint8 array of nbytes whose first byte lies `align` bytes past a 16-byte boundary."""
    raw = np.full(nbytes + 32, fill, np.uint8)
    start = (-raw.ctypes.data) % 16 + align
    return raw[start:start + nbytes]


def slot_bytes(bound):
    return (bound + 32 + 15) // 16 * 16


def well_formed(lo, hi, end, src_cap, bound):
    return end <= src_cap and 0 <= lo <= hi <= src_cap and hi - lo <= bound


def lift(src_addr, src_cap, src_off, bounds, cuts, seed=1):
    """Runs the step and the status step over the stages [b0, b1) of `cuts`.  Returns per stage (slot, so, sl, dc, io, out)."""
    n = len(bounds)
    src_off = np.asarray(src_off, np.int64)
    bounds = np.asarray(bounds, np.int32)
    got = []
    for b0, b1 in cuts:
        m = b1 - b0
        sizes = np.array([_lib().emu_lift_slot_bytes(int(b)) for b in bounds[b0:b1]], np.int64)
        assert list(sizes) == [slot_bytes(int(b)) for b in bounds[b0:b1]]
        slot = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        span = np.concatenate([src_off[b0:b1 + 1], src_off[n:n + 1]]).astype(np.int64)
        bound = bounds[b0:b1].copy()
        so, sl = slot[:m].copy(), np.full(m, -9, np.int32)
        dc, out = np.full(m, DC, np.int32), np.full(m, OUT, np.int32)
        io = _aligned(int(slot[m]) + 64, 0, IO_FILL)
        _lib().emu_lift_stage(src_addr, src_cap, slot.ctypes.data, span.ctypes.data, m, bound.ctypes.data, so.ctypes.data,
                              sl.ctypes.data, dc.ctypes.data, io.ctypes.data, out.ctypes.data, seed)
        got.append((slot, so, sl, dc, io, out))
    return got


def check(src_addr, src_bytes, src_cap, src_off, bounds, cuts, seed=1):
    """The contract, restated; src_bytes = the bytes at src_addr (at least src_cap of them).  Returns the rejected mask."""
    n = len(bounds)
    rejected = []
    for (b0, b1), (slot, so, sl, dc, io, out) in zip(cuts, lift(src_addr, src_cap, src_off, bounds, cuts, seed)):
        for k, i in enumerate(range(b0, b1)):
            lo, hi = int(src_off[i]), int(src_off[i + 1])
            ok = well_formed(lo, hi, int(src_off[n]), src_cap, int(bounds[i]))
            rejected.append(not ok)
            if ok:
                at = int(slot[k]) + (src_addr + lo) % 16
                assert so[k] == at and sl[k] == hi - lo and dc[k] == DC and out[k] == OUT, (i, lo, hi)
                assert bytes(io[at:at + hi - lo]) == bytes(src_bytes[lo:hi]), f"block {i}: staged bytes differ"
                assert at + hi - lo <= slot[k + 1] - 17, "less than the room the decoders read past a block"
            else:
                assert so[k] == slot[k] and sl[k] == 0 and dc[k] == 0 and out[k] == E_ARG, (i, lo, hi)
                assert (io[slot[k]:slot[k + 1]] == IO_FILL).all(), f"block {i}: a rejected block was staged"
        assert (io[slot[-1]:] == IO_FILL).all(), "written behind the last slot"
    return rejected


def _batch(lens, gaps, rng):
    """Blocks of `lens` bytes with `gaps` bytes before each, back to back: (bytes, src_off of n + 1 entries)."""
    off, pos = [], 0
    for l, g in zip(lens, gaps):
        pos += g
        off.append(pos)
        pos += l
    off.append(pos)
    return rng.integers(0, 256, pos + 64, dtype=np.uint8), np.array(off, np.int64)


@pytest.mark.parametrize("align", range(16))
def test_every_host_alignment_with_edge_block_sizes(align):
    rng = np.random.default_rng(200 + align)
    lens = [0, 1, 15, 16, 17, 65536, 3, 1, 1, 1, 2, 16]                   # several blocks inside one 16-byte unit
    data, off = _batch(lens, [0] * len(lens), rng)
    src = _aligned(len(data), align, 0)
    src[:] = data
    cap = int(off[-1])
    bounds = [l + l // 255 + 16 for l in lens]                             # compress_bound of a decode whose dst_cap = len
    for cuts in ([(0, len(lens))], [(0, 1), (1, 5), (5, 6), (6, 12)]):
        assert not any(check(src.ctypes.data, src, cap, off, bounds, cuts, seed=align + 1))


def test_a_block_of_exactly_its_bound_and_one_byte_over():
    rng = np.random.default_rng(5)
    for align in (0, 7, 15):
        lens = [40, 41, 8, 9, 100]
        data, off = _batch(lens, [3, 0, 1, 0, 2], rng)
        src = _aligned(len(data), align, 0)
        src[:] = data
        bounds = [40, 40, 8, 8, 100]                                       # an Unwrap's dst_cap + 8, say
        rej = check(src.ctypes.data, src, int(off[-1]), off, bounds, [(0, 2), (2, 5)])
        assert rej == [False, True, False, True, False]


def test_every_rejected_kind():
    rng = np.random.default_rng(9)
    data = rng.integers(0, 256, 4096, dtype=np.uint8)
    src = _aligned(len(data), 3, 0)
    src[:] = data
    cap = 1000
    # fine | decreasing | fine | decreasing | negative start | over its bound | past src_cap | starting past src_cap,
    # decreasing | empty, at src_cap
    off = np.array([0, 100, 50, 60, -5, 20, 700, 1001, 1000, 1000], np.int64)
    bounds = [200, 200, 200, 200, 200, 200, 400, 200, 200]
    want = [False, True, False, True, True, True, True, True, False]
    assert check(src.ctypes.data, src, cap, off, bounds, [(0, 4), (4, 9)]) == want
    assert check(src.ctypes.data, src, cap, off, bounds, [(0, 9)]) == want


def test_an_offload_that_did_not_fit_rejects_every_block():
    rng = np.random.default_rng(10)
    data, off = _batch([10, 20, 30], [0, 0, 0], rng)
    src = _aligned(len(data), 1, 0)
    src[:] = data
    for cap in (59, 30, 0):
        off2 = off.copy()
        off2[-1] = 60                                                      # src_off[n] > src_cap
        rej = check(src.ctypes.data, src, cap, off2, [100] * 3, [(0, 2), (2, 3)])
        assert all(rej)
    assert not any(check(src.ctypes.data, src, 60, off, [100] * 3, [(0, 2), (2, 3)]))


def test_random_batches_over_several_stages():
    rng = np.random.default_rng(21)
    for trial in range(8):
        n = int(rng.integers(1, 60))
        lens = [int(x) for x in rng.choice([0, 1, 2, 15, 16, 17, 31, 33, 100, 4096, 70000], n)]
        data, off = _batch(lens, [int(x) for x in rng.integers(0, 20, n)], rng)
        src = _aligned(len(data), int(rng.integers(0, 16)), 0)
        src[:] = data
        bounds = [int(l) + int(rng.integers(0, 50)) for l in np.diff(off)]          # a span holds the gap behind its block
        cuts, b0 = [], 0
        while b0 < n:
            b1 = min(n, b0 + int(rng.integers(1, 12)))
            cuts.append((b0, b1))
            b0 = b1
        assert not any(check(src.ctypes.data, src, int(off[-1]), off, bounds, cuts, seed=trial))


_FENCED = textwrap.dedent("""
    import ctypes as C, mmap, sys
    import numpy as np
    from tests import test_lift_host_emu as t
    a, b = int(sys.argv[1]), int(sys.argv[2])
    page = mmap.PAGESIZE
    libc = C.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    m = mmap.mmap(-1, 4 * page)
    base = C.addressof(C.c_char.from_buffer(m))
    # page 0 and page 3 are PROT_NONE; [src, src + cap) starts a bytes into page 1 and ends b bytes before page 3, so the
    # aligned units around it are exactly pages 1 and 2
    src_addr = base + page + a
    cap = 2 * page - a - b
    rng = np.random.default_rng(a * 16 + b)
    data = rng.integers(0, 256, cap, dtype=np.uint8)
    m[page + a:page + a + cap] = data.tobytes()
    assert libc.mprotect(base, page, 0) == 0 and libc.mprotect(base + 3 * page, page, 0) == 0
    big = cap + 16
    # the first block at 0, the last ending at src_cap; spans reaching past either end, and an offload that did not fit
    off = np.array([0, 1, 17, 600, 2000, cap - 1, cap, cap], np.int64)
    t.check(src_addr, data, cap, off, [big] * 7, [(0, 3), (3, 7)])
    for bad in ([0, cap + 1, cap + 1], [-1, 5, cap], [cap - 3, cap + 15, cap + 15], [-16, -1, cap], [cap, cap + 16, cap]):
        off = np.array(bad, np.int64)
        rej = t.check(src_addr, data, cap, off, [big] * 2, [(0, 2)])
        assert any(rej), bad
    off = np.array([0, 100, cap + 1], np.int64)
    assert all(t.check(src_addr, data, cap, off, [big] * 2, [(0, 1), (1, 2)]))
    print("ok")
""")


@pytest.mark.parametrize("a,b", [(0, 0), (1, 0), (0, 1), (15, 15), (7, 9), (3, 14)])
def test_nothing_outside_the_aligned_units_around_src_is_read(a, b):
    _lib()                                                                 # build here, so the child only loads it
    r = subprocess.run([sys.executable, "-c", _FENCED, str(a), str(b)], cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip() == "ok", (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
