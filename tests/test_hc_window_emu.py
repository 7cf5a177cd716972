"""LZ4HC for blocks above 64 KiB, one warp per block over a sliding 64 KiB window (lz4net_b200/csrc/lz4hc_window.cuh), on
the CPU warp emulator.  A block either gets the reference's (result, bytes) or is handed back (HCW_FALLBACK), nothing
else."""
import numpy as np
import pytest

import oracle
from tests import cases
from tests import emu_hcw_window as win

FB = win.HCW_FALLBACK


def _check(d, cap=None, **kw):
    """True = encoded like the reference, False = handed back."""
    r, o = win.encode(d, cap=cap, **kw)
    if r == FB:
        return False
    assert (r, o) == oracle.encode_hc(d, cap=cap), (len(d), cap, kw)
    return True


def _rand(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


# every model at the sizes around the segment boundaries; the emulator needs seconds per 64 KiB on the dense models, so
# each model takes two of the sizes and only the fast ones take a whole MiB
SIZES = (65537, 65547, 131071, 131072, 131073, 200003)


@pytest.mark.parametrize("model", cases.MODELS)
def test_window_corpus_matches_oracle(model):
    i = cases.MODELS.index(model)
    sizes = [SIZES[i % len(SIZES)], SIZES[(i + 3) % len(SIZES)]]
    if model in ("lowent", "ETEXT"):                                   # the slowest to emulate: one block, just past 64 KiB
        sizes = [65547 if model == "lowent" else 131073]
    if model in ("E100", "periodic", "runs"):
        sizes.append(1 << 20)
    for n in sizes:
        d = cases.content(model, n, seed=70 + n).tobytes()
        assert _check(d, sched_seed=n % 97 + 1), (model, n)


def _plant(n, marks, seed=1):
    """Random bytes (no 4-byte string repeats by chance) with the same 12-byte string at every position in `marks`."""
    d = bytearray(_rand(n, seed))
    s = b"\x01WINDOWEDGE\x02"
    for p in marks:
        d[p:p + len(s)] = s
    return bytes(d)


@pytest.mark.parametrize("q", [65536 + 40, 131072, 131072 + 3, 196608 - 1, 196608 + 17])
def test_window_edges(q):
    """A candidate exactly 65535 back is taken, one 65536 back is not; a bucket whose previous position lies 65535 / 65536
    back (the reference clamps that delta); each with q on and across a segment boundary."""
    n = q + 5000
    for marks in ([q - 65535, q], [q - 65536, q], [q - 65536 - 65535, q - 65536, q], [q - 65536 - 65536, q - 65536, q],
                  [q - 65536 - 1, q - 1, q], [q - 70000, q - 65535, q - 65534, q]):
        if min(marks) >= 1:
            assert _check(_plant(n, marks, seed=q)), (q, marks)


@pytest.mark.parametrize("q", [65535, 65536])
def test_window_position_zero(q):
    """q <= 65535 with an empty bucket: position 0 is the walk's last candidate; from 65536 on it is out of the window."""
    d = bytearray(_rand(q + 3000, q))
    d[0:12] = d[q:q + 12] = b"\x03ZEROWINDOW\x04"
    assert _check(bytes(d))


def test_window_long_matches_skip_segments():
    """Runs of 100-300 KiB inside text: one match jumps one or several segments, which are never indexed."""
    t = cases.content("mixed", 30000, seed=5).tobytes()
    for run in (100_000, 300_000):
        d = t + bytes(run) + t[::-1] + bytes([7]) * (run // 2) + t
        assert _check(d), run


def test_window_repeat_detector_runs_longer_than_a_segment():
    for m, n in (("E100", 140000), ("runs", 150000), ("periodic", 131075)):
        assert _check(cases.content(m, n, seed=21).tobytes()), (m, n)
    for period in (1, 2, 3, 4):
        d = _rand(3000, period) + bytes(range(10, 10 + period)) * (200000 // period) + _rand(3000, period + 9)
        assert _check(d), period


def test_window_one_bucket_holds_a_whole_segment():
    """Zeros over three segments: a bucket end of 65536, a segment whose counters all sit in one bucket."""
    assert _check(bytes(196608 + 4000))
    assert _check(bytes(200000) + cases.content("mixed", 5000, seed=3).tobytes())


def _hash15(b4):
    return ((int.from_bytes(b4, "little") * 2654435761) & 0xFFFFFFFF) >> 17


def test_window_hands_back_the_colliding_triple():
    """A run of period 3 two of whose strings share a hash bucket, past 64 KiB: the repeat detector's chain is not the
    static one, so the block is handed back (and the same run with a triple that does not collide is encoded)."""
    found = None
    for a in range(1, 256):
        for b in range(a + 1, 256):
            for c in range(b + 1, 256):
                s0, s1, s2 = bytes([a, b, c, a]), bytes([b, c, a, b]), bytes([c, a, b, c])
                if _hash15(s1) == _hash15(s2) and _hash15(s0) != _hash15(s1):
                    found = (a, b, c); break
            if found: break
        if found: break
    d = _rand(70000, 3) + bytes(found) * 200 + _rand(500, 4)
    assert win.encode(d)[0] == FB
    assert _check(_rand(70000, 3) + bytes([1, 2, 3]) * 200 + _rand(500, 4))


def test_window_limited_output():
    """Capacities from nothing to the bound on a block above 64 KiB: the limit checks of :529 / :541 / :731 fail at the
    start, in the middle and at the end of the output."""
    d = cases.content("mixed", 66000, seed=8).tobytes()
    r, _ = oracle.encode_hc(d)
    rng = np.random.default_rng(4)
    caps = set(range(0, 24)) | set(range(r - 24, r + 3)) | {int(c) for c in rng.integers(24, r - 24, 24)}
    for cap in sorted(caps):
        assert _check(d, cap=cap), cap


def test_window_alignment_and_lane_schedules():
    d = cases.content("mixed", 70001, seed=12).tobytes()
    for skew in (1, 2, 3, 7, 13):
        assert _check(d, src_skew=skew, dst_skew=(skew * 5) % 16, sched_seed=skew), skew
    for seed in (2, 99, 12345):
        assert _check(d, sched_seed=seed), seed


@pytest.mark.parametrize("behind", [True, False])
def test_window_reads_no_word_outside_the_block(behind):
    """A PROT_NONE page directly behind the block's last byte / in front of its first: no word without an input byte is read."""
    for n in (65537, 131074):
        d = cases.content("mixed", n, seed=n).tobytes()
        assert win.encode_fenced(d, behind=behind) == oracle.encode_hc(d), (n, behind)
