"""The per-thread rules of the asynchronous LZ4Stream calls (lz4_stream.cuh) on the CPU warp emulator.

lz4b200_stream_encode_from_device_async holds no per-chunk host metadata: each pipeline stage's chunk table (source
offset, length, dense slot offset, capacity) is computed on the device from the stage's first chunk, its chunk count, the
chunk size and the stream's length.  lz4b200_stream_decode_to_device_async keeps its status on the device: after each
stage a kernel sets the call's failure flag when a compressed chunk's decode did not read exactly its compLen bytes.  Here
both rules run on the emulator against the host formulas."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import emu

_P, _I32, _I64, _U64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
_alib = None


def _lib():
    """The rules' harness unit (tests/simt_emu/emu_stream_async.cpp), built by the emulator driver's builder."""
    global _alib
    if _alib is None:
        l = C.CDLL(emu.build(os.path.join(os.path.dirname(os.path.abspath(emu.__file__)), "simt_emu", "emu_stream_async.cpp")))
        l.emu_stream_cut.restype = None
        l.emu_stream_cut.argtypes = [_I64, _I32, _I32, _I64, _P, _P, _P, _P, _U64]
        l.emu_stream_status.restype = C.c_int
        l.emu_stream_status.argtypes = [_I32, _P, _P, _P, _P, _U64]
        _alib = l
    return _alib


def _cut(first, m, block_size, n, seed=1):
    so, dof = np.full(m + 4, -7, np.int64), np.full(m + 4, -7, np.int64)
    ln, cap = np.full(m + 4, -7, np.int32), np.full(m + 4, -7, np.int32)
    _lib().emu_stream_cut(first, m, block_size, n, so.ctypes.data, ln.ctypes.data, dof.ctypes.data, cap.ctypes.data, seed)
    for a in (so, dof, ln, cap):
        assert (a[m:] == -7).all(), "the rule wrote behind the stage's m entries"
    return so[:m], ln[:m], dof[:m], cap[:m]


def _host_cut(first, m, block_size, n):
    """The host formula: chunk i is bytes [i * block_size, min((i + 1) * block_size, n)); its slot starts at the sum of the
    stage's earlier capacities."""
    so = (first + np.arange(m, dtype=np.int64)) * block_size
    ln = np.minimum(block_size, n - so).astype(np.int32)
    dof = np.concatenate([[0], np.cumsum(ln.astype(np.int64))[:-1]]) if m else np.zeros(0, np.int64)
    return so, ln, dof, ln


def _stages(n, block_size, per):
    """The stage plan of an asynchronous encode: per chunks a stage, the last one short."""
    chunks = (n + block_size - 1) // block_size
    return [(k0, min(per, chunks - k0)) for k0 in range(0, chunks, per)]


def _check(n, block_size, per, seed=1):
    covered = 0
    for first, m in _stages(n, block_size, per):
        got, want = _cut(first, m, block_size, n, seed), _host_cut(first, m, block_size, n)
        for g, w, what in zip(got, want, ("so", "len", "dof", "cap")):
            assert (g == w).all(), (n, block_size, first, m, what)
        covered += int(got[1].astype(np.int64).sum())
        assert (got[1] >= 1).all() and (got[1] <= block_size).all()
    assert covered == n                                                 # the stages cover the stream exactly once


@pytest.mark.parametrize("n,block_size,per", [
    (1, 1, 1), (17, 1, 5), (100, 7, 3), (100, 100, 1), (100, 101, 4), (5, 1 << 20, 1),
    ((1 << 20) + 3, 4096, 64), (3 * 65536 - 1, 65536, 2), (1000, 16, 1 << 20),
    ((1 << 31) + 5, (1 << 31) - 12, 1),                                 # chunks near the largest a frame may hold
])
def test_chunk_table_edges(n, block_size, per):
    """A final partial chunk, block_size > n, block_size = 1, one chunk a stage, and chunk counts crossing many stages."""
    _check(n, block_size, per)


def test_chunk_table_random():
    rng = np.random.default_rng(20)
    for t in range(300):
        block_size = int(rng.choice([1, 2, 3, 16, 100, 4096, 65536, 65537, 1 << 20, int(rng.integers(1, 1 << 22))]))
        n = int(rng.integers(1, 64)) * block_size + int(rng.integers(-min(block_size - 1, 5000), min(block_size, 5000)))
        n = max(n, 1)
        per = int(rng.integers(1, 80))
        _check(n, block_size, per, seed=t)


def test_chunk_table_far_into_a_large_stream():
    """A stage far into a stream whose byte offsets pass 2^32 (so in int64, chunk index * block_size)."""
    bs, first, m = 4096, (1 << 21) + 3, 70
    n = (first + m) * bs - 11
    got, want = _cut(first, m, bs, n), _host_cut(first, m, bs, n)
    for g, w in zip(got, want):
        assert (g == w).all()
    assert got[1][-1] == bs - 11


def _status(stages, comp_len, stored, res, seed=1):
    m = np.array([len(s) for s in stages], np.int32)
    c, s, r = (np.ascontiguousarray(a, np.int32) for a in (comp_len, stored, res))      # kept alive across the call
    return _lib().emu_stream_status(len(stages), m.ctypes.data, c.ctypes.data, s.ctypes.data, r.ctypes.data, seed)


def _host_failed(comp_len, stored, res):
    return int(any(s == 0 and r != c for c, s, r in zip(comp_len, stored, res)))


def test_status_rule_random():
    """The flag is set exactly when some compressed entry's result differs from its compLen, negative results included;
    stored entries (their stored length > 0: the decoder got a neutral entry, whatever it returned) never set it."""
    rng = np.random.default_rng(21)
    for t in range(400):
        sizes = [int(x) for x in rng.integers(0, 70, int(rng.integers(1, 6)))]
        total = sum(sizes)
        comp_len = rng.integers(1, 1 << 20, total).astype(np.int32)
        stored = np.where(rng.random(total) < 0.3, rng.integers(1, 1 << 20, total), 0).astype(np.int32)
        res = comp_len.copy()
        # the neutral entry of a stored chunk decodes to anything; a compressed one fails now and then
        res[stored > 0] = rng.integers(-(1 << 20), 1 << 20, int((stored > 0).sum()))
        bad = (rng.random(total) < (0.02 if t % 3 else 0.0)) & (stored == 0)
        res[bad] = np.where(rng.random(int(bad.sum())) < 0.5, -rng.integers(1, 1 << 20, int(bad.sum())),
                            comp_len[bad] + rng.integers(1, 9, int(bad.sum())) * rng.choice([-1, 1], int(bad.sum())))
        stages = [list(range(s)) for s in sizes]
        assert _status(stages, comp_len, stored, res, seed=t) == _host_failed(comp_len, stored, res), t


@pytest.mark.parametrize("case,stored,res,want", [
    ("all-ok", [0, 0, 5], [10, 20, -1], 0),
    ("compressed-short-read", [0, 0, 0], [10, 19, 30], 1),
    ("compressed-negative", [0, 0, 0], [10, -5, 30], 1),
    ("compressed-long-read", [0, 0, 0], [10, 20, 31], 1),
    ("stored-negative-ignored", [7, 7, 7], [-1, -1, -1], 0),
    ("stored-mismatch-ignored", [0, 9, 0], [10, 3, 30], 0),
])
def test_status_rule_cases(case, stored, res, want):
    assert _status([[0, 1, 2]], [10, 20, 30], stored, res) == want, case


def test_status_rule_empty_stages_and_late_failure():
    """Empty stages are passed over; a failure in the last of many stages still sets the flag; none sets it for none."""
    assert _status([[], [], []], [], [], []) == 0
    assert _status([[0], [], [0, 1]], [4, 5, 6], [0, 0, 0], [4, 5, 6]) == 0
    comp = np.arange(1, 201, dtype=np.int32)
    res = comp.copy()
    res[-1] = 0
    stages = [list(range(50))] * 4
    assert _status(stages, comp, np.zeros(200, np.int32), res) == 1
