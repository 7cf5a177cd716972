"""LZ4HC for blocks above 64 KiB, one warp per block over a sliding 64 KiB window (lz4net_b200/csrc/lz4hc_window.cuh), on
the CPU warp emulator.  A block either gets the reference's (result, bytes) or is handed back (HCW_FALLBACK), nothing
else.  The planted blocks are tests/hcedge.py's window cases, which the H100 tests run too; each says which of the two
the window kernel must do, and the thread kernel must give the reference's bytes on every one."""
import numpy as np
import pytest

import oracle
from tests import cases, emu, hcedge

FB = emu.HCW_FALLBACK


def _check(d, cap=None, **kw):
    """True = encoded like the reference, False = handed back."""
    r, o = emu.encode_hcw_window(d, cap=cap, **kw)
    if r == FB:
        return False
    assert (r, o) == oracle.encode_hc(d, cap=cap), (len(d), cap, kw)
    return True


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


def _planted(prefix):
    """Runs tests/hcedge.py's window cases whose names start with `prefix` through the window and the thread kernel."""
    got = [c for c in hcedge.window_cases(1) if c.name.startswith(prefix)]
    assert got, prefix
    for i, c in enumerate(got):
        want = oracle.encode_hc(c.data)
        assert emu.encode_hc(c.data) == want, c.name
        r, o = emu.encode_hcw_window(c.data, sched_seed=i + 1)
        assert (r, o) == want if c.warp else r == FB, c.name


@pytest.mark.parametrize("q", hcedge.WINDOW_Q)
def test_window_edges(q):
    """A candidate exactly 65535 back is taken, one 65536 back is not; a bucket whose previous position lies 65535 / 65536
    back (the reference clamps that delta); each with q on and across a segment boundary."""
    _planted(f"window-q{q}-")


@pytest.mark.parametrize("q", [65535, 65536])
def test_window_position_zero(q):
    """q <= 65535 with an empty bucket: position 0 is the walk's last candidate; from 65536 on it is out of the window."""
    _planted(f"window-pos0-q{q}")


def test_window_long_matches_skip_segments():
    """Runs of 100-300 KiB inside text: one match jumps one or several segments, which are never indexed."""
    _planted("window-skip-")


def test_window_repeat_detector_runs_longer_than_a_segment():
    for m, n in (("E100", 140000), ("runs", 150000), ("periodic", 131075)):
        assert _check(cases.content(m, n, seed=21).tobytes()), (m, n)
    _planted("window-repeat-period")


def test_window_one_bucket_holds_a_whole_segment():
    """Zeros over three segments: a bucket end of 65536, a segment whose counters all sit in one bucket."""
    _planted("window-one-bucket-")


def test_window_hands_back_the_colliding_triple():
    """A run of period 3 two of whose strings share a hash bucket, past 64 KiB: the repeat detector's chain is not the
    static one, so the block is handed back (and the same run with a triple that does not collide is encoded)."""
    _planted("window-colliding-triple")
    _planted("window-triple-not-colliding")


def test_window_limited_output_planted():
    """Capacities around the start and the end of the output over a planted block whose one long match is 65535 back."""
    d = next(c for c in hcedge.window_cases(1) if c.name == "window-q131072-65535").data
    r, _ = oracle.encode_hc(d)
    for cap in sorted({0, 1, 2, 15, 16, 17, 270, 4096, 65535, 65536, len(d), r - 3, r - 2, r - 1, r, r + 1}):
        assert _check(d, cap=cap), cap


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
        assert emu.encode_hcw_window(d, fence="behind" if behind else "front") == oracle.encode_hc(d), (n, behind)
