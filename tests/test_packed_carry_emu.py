"""The placement step of the packed decodes (lz4_packed.cuh) on the CPU warp emulator.

lz4b200_decode_batch_packed_to_device decodes a batch a pipeline stage at a time: each stage measures its blocks, scans the
sizes, and this step places the blocks behind the earlier stages' (the running total carried from stage to stage) and sets
the flag its decoders run behind.  Here the step itself runs on the emulator, chained by hand the way the pipeline chains
it through its cells, against a NumPy restatement of the contract: offsets = the exclusive prefix sum of max(size, 0) over
the whole batch, capacities = max(size, 0), a stage fits exactly when everything up to its end fits."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import emu

_P, _I, _L, _U64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
_plib = None
NSLOT = 3
I32_MAX = 2 ** 31 - 1


def _lib():
    """The step's harness unit (tests/simt_emu/emu_packed.cpp), built by the emulator driver's builder."""
    global _plib
    if _plib is None:
        l = C.CDLL(emu.build(os.path.join(os.path.dirname(os.path.abspath(emu.__file__)), "simt_emu", "emu_packed.cpp")))
        l.emu_packed_place.restype = None
        l.emu_packed_place.argtypes = [_P, _P, _I, _P, _L, _P, _P, _P, _P, _U64]
        _plib = l
    return _plib


def _scan(sizes):
    """What the scan leaves for a stage: int64[m+1], the exclusive prefix sum of max(size, 0) and the stage's total."""
    return np.concatenate([[0], np.cumsum(np.maximum(sizes, 0), dtype=np.int64)]).astype(np.int64)


def _pipeline(stages, total_cap, seed=1):
    """The stages' steps in order, the running total in NSLOT cells as the pipeline keeps it: stage k reads the cell of
    stage k-1 (the first reads none) and writes its own.  Returns per stage (abs_off, cap, fits, total)."""
    cells = np.full(NSLOT, -12345, np.int64)
    out = []
    for k, sizes in enumerate(stages):
        sizes = np.asarray(sizes, np.int32)
        m = len(sizes)
        off = _scan(sizes)
        cap = np.full(m + 1, -77, np.int32)
        abs_off = np.full(m + 1, -77, np.int64)
        fits = np.full(1, -77, np.int32)
        base_in = cells[(k - 1) % NSLOT:].ctypes.data if k else None
        _lib().emu_packed_place(sizes.ctypes.data, off.ctypes.data, m, base_in, total_cap, cap.ctypes.data, abs_off.ctypes.data,
                                fits.ctypes.data, cells[k % NSLOT:].ctypes.data, seed + k)
        assert cap[m] == -77 and abs_off[m] == -77, "the step wrote behind its m entries"
        assert fits[0] in (0, 1)
        out.append((abs_off[:m].copy(), cap[:m].copy(), int(fits[0]), int(cells[k % NSLOT])))
    return out


def _want(stages, total_cap):
    """The contract, over the whole batch at once."""
    flat = np.concatenate([np.asarray(s, np.int64) for s in stages]) if stages else np.zeros(0, np.int64)
    off = np.concatenate([[0], np.cumsum(np.maximum(flat, 0))])
    out, i = [], 0
    for s in stages:
        m = len(s)
        end = int(off[i + m])
        out.append((off[i:i + m], np.maximum(np.asarray(s, np.int64), 0), int(end <= total_cap), end))
        i += m
    return out


def _check(stages, total_cap, seed=1):
    got, want = _pipeline(stages, total_cap, seed), _want(stages, total_cap)
    for k, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]) and g[2:] == w[2:], (k, total_cap)
    fits = [g[2] for g in got]
    assert fits == sorted(fits, reverse=True), "a stage behind one that does not fit fits"
    return got


def test_stages_chain_like_one_scan_over_the_batch():
    rng = np.random.default_rng(5)
    for trial in range(40):
        stages = [rng.integers(-6, 70000, int(rng.integers(1, 200))).astype(np.int32) for _ in range(int(rng.integers(1, 12)))]
        total = sum(int(np.maximum(s, 0).sum()) for s in stages)
        for cap in (total, total - 1, total // 2, 0, total + 1000):
            _check(stages, cap, seed=trial + 1)


def test_negative_sizes_occupy_nothing_and_empty_stages_pass_the_total_on():
    stages = [[-1, -5, 10, -1], [], [-3, -3], [0, 0, 0], [], [7], [-2 ** 31, I32_MAX]]
    got = _check(stages, 10 + 7 + I32_MAX)
    assert [g[3] for g in got] == [10, 10, 10, 10, 10, 17, 17 + I32_MAX]
    assert got[0][1].tolist() == [0, 0, 10, 0] and got[0][0].tolist() == [0, 0, 0, 10]
    assert got[6][1].tolist() == [0, I32_MAX] and got[6][0].tolist() == [17, 17]
    assert all(g[2] == 1 for g in got)


def test_a_stage_of_more_than_one_warp_and_of_one_block():
    stages = [[3] * 33, [5], [2] * 1000, [1]]
    _check(stages, 99 + 5 + 2000 + 1)
    _check(stages, 99 + 5 + 2000)


def test_the_running_total_crosses_2_31_and_2_32():
    stages = [[I32_MAX, 1], [I32_MAX, -4, I32_MAX], [100], [I32_MAX] * 5]
    total = 8 * I32_MAX + 101
    got = _check(stages, total)
    assert got[0][3] == 2 ** 31 and got[1][0].tolist() == [2 ** 31, 2 ** 32 - 1, 2 ** 32 - 1] and got[1][3] == 3 * 2 ** 31 - 2
    assert got[3][3] == total and all(g[2] == 1 for g in got)
    for cap in (2 ** 31 - 1, 2 ** 31, 2 ** 32 - 2, 2 ** 32 + 98, 2 ** 32 + 99):
        _check(stages, cap)


def test_the_flag_flips_exactly_where_the_total_passes_the_capacity():
    stages = [[10, 20], [30], [40, -1, 50]]
    ends = [30, 60, 150]
    for k, end in enumerate(ends):
        fits = [g[2] for g in _check(stages, end)]                  # total up to stage k == cap: it fits, the next does not
        assert fits == [1] * (k + 1) + [0] * (2 - k)
        fits = [g[2] for g in _check(stages, end - 1)]              # one byte short: stage k does not fit any more
        assert fits == [1] * k + [0] * (3 - k)
    assert [g[2] for g in _check(stages, 0)] == [0, 0, 0]
    assert [g[2] for g in _check([[0], [-1], []], 0)] == [1, 1, 1]  # an empty total fits an empty destination


def test_a_stage_that_does_not_fit_still_reports_offsets_and_total():
    """The caller learns the needed total from a call that did not fit: offsets and the running total do not depend on the
    capacity."""
    stages = [[100, 200], [300], [-9, 400]]
    a, b = _pipeline(stages, 0), _pipeline(stages, 10 ** 12)
    for x, y in zip(a, b):
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]) and x[3] == y[3]
    assert a[-1][3] == 1000 and [x[2] for x in a] == [0, 0, 0] and [y[2] for y in b] == [1, 1, 1]


@pytest.mark.parametrize("n", [1, 31, 32, 257])
def test_a_batch_in_one_piece_gets_capacities_and_the_flag_only(n):
    """lz4b200_decode_batch_packed and lz4b200_unwrap_batch_packed run the step without a base, absolute offsets or a total:
    capacity = max(size, 0), fits = off[n] <= total_cap, nothing else is written."""
    sizes = np.random.default_rng(n).integers(-5, 5000, n).astype(np.int32)
    off = _scan(sizes)
    for total_cap, want in ((int(off[n]), 1), (int(off[n]) - 1, 0), (int(off[n]) + 1, 1)):
        cap = np.full(n + 1, -77, np.int32)
        fits = np.full(1, -77, np.int32)
        _lib().emu_packed_place(sizes.ctypes.data, off.ctypes.data, n, None, total_cap, cap.ctypes.data, None, fits.ctypes.data,
                                None, 3)
        assert cap[:n].tolist() == np.maximum(sizes, 0).tolist() and cap[n] == -77 and fits[0] == want
