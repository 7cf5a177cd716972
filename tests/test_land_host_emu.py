"""The landing step of the asynchronous packed encode into page-locked host memory (lz4_land.cuh) on the CPU warp emulator.

lz4b200_encode_batch_packed_from_device_async encodes a batch a pipeline stage at a time into dense device slots, scans
the lengths, and this step writes the stage's offsets, lengths and running total and moves its bytes to where they land in
the caller's host memory, gathered by 16-byte output unit.  Here the step runs on the emulator over real host buffers,
chained by hand through two carry cells the way the pipeline chains it, against a NumPy restatement of the contract: the
destination holds the blocks back to back, out_off is the exclusive prefix sum over the whole batch, a stage lands exactly
when everything up to its end fits, and nothing in front of the destination or behind its capacity is written."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import emu

_P, _I, _L, _U64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
_llib = None
NASYNC = 2                                                               # the context's asynchronous stage buffers
CANARY = 0xC3
GUARD = 48                                                               # canary bytes in front of dst and behind its capacity


def _lib():
    """The step's harness unit (tests/simt_emu/emu_land.cpp), built by the emulator driver's builder."""
    global _llib
    if _llib is None:
        l = C.CDLL(emu.build(os.path.join(os.path.dirname(os.path.abspath(emu.__file__)), "simt_emu", "emu_land.cpp")))
        l.emu_land_stage.restype = None
        l.emu_land_stage.argtypes = [_P, _P, _P, _P, _I, _P, _L, _P, _P, _P, _P, _U64]
        _llib = l
    return _llib


def _aligned(nbytes, align, fill):
    """A uint8 array of nbytes whose first byte lies `align` bytes past a 16-byte boundary (and the buffer keeping it)."""
    raw = np.full(nbytes + 32, fill, np.uint8)
    start = (-raw.ctypes.data) % 16 + align
    return raw[start:start + nbytes]


def _land(stages, total_cap, align, rng, seed=1):
    """Runs the stages' steps in order.  stages: lists of block lengths.  Returns (dst with its guards, blocks, out_off,
    out_len, per-stage running totals)."""
    n = sum(len(s) for s in stages)
    blocks = [rng.integers(0, 256, l, dtype=np.uint8) for s in stages for l in s]
    buf = _aligned(GUARD + max(total_cap, 0) + GUARD, align, CANARY)      # dst = buf[GUARD:]
    dst_addr = buf.ctypes.data + GUARD
    out_off, out_len = np.full(n + 1, -7, np.int64), np.full(n, 12345, np.int32)
    cells = np.full(NASYNC, -12345, np.int64)
    totals, b0 = [], 0
    for k, lens in enumerate(stages):
        m = len(lens)
        lens = np.asarray(lens, np.int32)
        # the stage's dense slots: each block in a slot of its capacity (the encoder's bound, or more), the room behind its
        # bytes and the buffer's 64-byte tail holding garbage that must never land
        caps = lens.astype(np.int64) + rng.integers(0, 40, m)
        dof = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64) if m else np.zeros(0, np.int64)
        dense = _aligned(int(caps.sum()) + 64, 0, 0)
        dense[:] = rng.integers(0, 256, dense.size, dtype=np.uint8)
        for i in range(m):
            dense[dof[i]:dof[i] + lens[i]] = blocks[b0 + i]
        off = np.concatenate([[0], np.cumsum(lens, dtype=np.int64)]).astype(np.int64)
        base_in = cells[(k - 1) % NASYNC:].ctypes.data if k else None
        _lib().emu_land_stage(dense.ctypes.data, dof.ctypes.data, lens.ctypes.data, off.ctypes.data, m, base_in, total_cap,
                              dst_addr, out_off[b0:].ctypes.data, out_len[b0:].ctypes.data, cells[k % NASYNC:].ctypes.data,
                              seed + k)
        totals.append(int(cells[k % NASYNC]))
        b0 += m
    return buf, blocks, out_off, out_len, totals


def _check(stages, total_cap, align, rng, seed=1):
    buf, blocks, out_off, out_len, totals = _land(stages, total_cap, align, rng, seed)
    lens = np.array([len(b) for b in blocks], np.int64)
    want_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n = len(blocks)
    assert np.array_equal(out_off, want_off), "out_off is not the exclusive prefix sum over the batch"
    assert np.array_equal(out_len, lens.astype(np.int32))
    ends, b0 = [], 0
    for s in stages:
        b0 += len(s)
        ends.append(int(want_off[b0]))
    assert totals == ends
    # a stage lands exactly when everything up to its end fits; the running total never shrinks, so the landed stages
    # are a prefix of the batch and everything behind them keeps its canary
    landed = max([e for e in ends if e <= total_cap], default=0)
    concat = np.concatenate(blocks) if n else np.zeros(0, np.uint8)
    assert (buf[:GUARD] == CANARY).all(), "written in front of dst"
    dst = buf[GUARD:]
    assert np.array_equal(dst[:landed], concat[:landed]), "landed bytes differ from the blocks back to back"
    assert (dst[landed:] == CANARY).all(), "written behind the landed stages or behind dst_total_cap"
    return landed, ends


@pytest.mark.parametrize("align", range(16))
def test_every_base_alignment_with_edge_block_sizes(align):
    rng = np.random.default_rng(100 + align)
    sizes = [0, 1, 15, 16, 17, 65536 + 37]
    for trial in range(3):
        stages = [list(rng.choice(sizes, int(rng.integers(1, 7)))) for _ in range(int(rng.integers(1, 6)))]
        total = sum(sum(s) for s in stages)
        _, ends = _check(stages, total, align, rng, seed=trial + 1)
        assert ends[-1] == total


def test_random_layouts_and_a_stage_whose_end_crosses_the_capacity():
    rng = np.random.default_rng(7)
    for trial in range(12):
        stages = [[int(x) for x in rng.choice([0, 1, 2, 3, 15, 16, 17, 31, 33, 100, 4096, 70000], int(rng.integers(0, 9)))]
                  for _ in range(int(rng.integers(1, 7)))]
        total = sum(sum(s) for s in stages)
        ends = np.cumsum([sum(s) for s in stages])
        k = int(rng.integers(0, len(stages)))
        inside = int(ends[k]) - int(rng.integers(1, max(sum(stages[k]), 1) + 1)) if sum(stages[k]) else int(ends[k])
        for cap in (total, total - 1, inside, 0, total + 17):
            if cap >= 0:
                _check(stages, cap, int(rng.integers(0, 16)), rng, seed=trial)


def test_a_stage_that_does_not_fit_still_reports_offsets_lengths_and_total():
    rng = np.random.default_rng(3)
    stages = [[100, 200], [300], [0, 400]]
    for cap, landed in ((1000, 1000), (999, 600), (600, 600), (599, 300), (300, 300), (0, 0)):
        got, ends = _check(stages, cap, 5, rng)
        assert got == landed and ends == [300, 600, 1000]


def test_many_one_byte_blocks_inside_one_unit():
    """Sixteen or fewer blocks of one byte (and empty ones between them) share a unit, and stages share its edges."""
    rng = np.random.default_rng(11)
    for align in range(16):
        stages = [[1, 0, 1, 1], [1] * 5, [0], [1, 1, 0, 0, 1], [1] * 9, [1, 1]]
        _check(stages, sum(map(sum, stages)), align, rng, seed=align)
        _check([[1] * 40], 40, align, rng, seed=align)


def test_empty_stages_and_an_empty_batch_pass_the_total_on():
    rng = np.random.default_rng(13)
    _, ends = _check([[0, 0], [], [5], [], [0]], 5, 9, rng)
    assert ends == [0, 0, 5, 5, 5]
    _, ends = _check([[0]], 0, 0, rng)
    assert ends == [0]


def test_a_stage_of_more_than_one_warp_of_units_and_entries():
    rng = np.random.default_rng(17)
    stages = [[17] * 100, [1] * 70, [65536 + 1, 3], [16] * 33]
    total = sum(map(sum, stages))
    for cap in (total, total - 1):
        _check(stages, cap, 3, rng)
