"""The LZ4HC kernels on constructed blocks (tests/hcedge.py) on the CPU warp emulator: the thread kernel
(lz4hc_encode.cuh), the warp kernel in both placements (lz4hc_warp.cuh) and the window kernel (lz4hc_window.cuh) against
the oracle, at the ends of the attempt budget in the search and the literal scan, at position 0, on ties, at matchlimit,
around the warp count's 128-byte steps, on backward extensions and repeats.  Each case says whether the warp kernels
encode it or hand it back, and they must do exactly that: the warp path, not the fallback, is what these blocks test.
The catalogue's blocks above 64 KiB run through the window and the thread kernel in tests/test_hc_window_emu.py."""
import pytest

import oracle
from tests import emu, hcedge

FB = emu.HCW_FALLBACK


@pytest.fixture(scope="module")
def catalogue():
    return [c for c in hcedge.catalogue(1) if len(c.data) <= 65536]


def test_catalogue_covers_the_edges():
    full = hcedge.catalogue(1)
    names = [c.name for c in full]
    for prefix, count in (("search-budget-place", 15), ("search-budget-repeat-", 2), ("scan-budget-", 5), ("pos0-", 8),
                          ("tie-search-", 14), ("tie-wider-", 4), ("forward-", 18), ("matchlimit-", 32),
                          ("back-limit-", 12), ("back-ref0-", 12), ("repeat-period", 24), ("window-q", 26), ("window-pos0-", 2), ("window-skip-", 2),
                          ("window-one-bucket-", 2), ("window-repeat-period", 4), ("window-", 38)):
        assert sum(n.startswith(prefix) for n in names) == count, prefix
    assert sum(not c.warp for c in full) == 3
    assert len(full) <= 300 and sum(len(c.data) <= 8192 for c in full) >= 140


def test_thread_kernel_matches_the_oracle(catalogue):
    for i, c in enumerate(catalogue):
        assert emu.encode_hc(c.data, src_skew=i % 4) == oracle.encode_hc(c.data), c.name


@pytest.mark.parametrize("smem", [True, False], ids=["smem", "l1"])
def test_warp_kernels_match_the_oracle(catalogue, smem):
    """Every case at a lane schedule and source / destination skew of its own; a block the case says the warp kernels
    encode must come out as the reference's bytes, one they hand back must be handed back."""
    for i, c in enumerate(catalogue):
        r, o = emu.encode_hcw(c.data, sched_seed=3 + 7 * i + smem, src_skew=(i + smem) % 16, dst_skew=(5 * i) % 16,
                              smem=smem)
        if c.warp:
            assert (r, o) == oracle.encode_hc(c.data), c.name
        else:
            assert r == FB, c.name


@pytest.mark.parametrize("sched", [1, 99, 12345])
def test_warp_kernel_lane_schedules(catalogue, sched):
    """The budget, position-0 and tie cases under more lane schedules (the order in which lanes run between votes)."""
    for c in catalogue:
        if c.name.startswith(("search-budget", "scan-budget", "pos0-", "tie-")):
            assert emu.encode_hcw(c.data, sched_seed=sched, smem=sched % 2 == 1) == oracle.encode_hc(c.data), (c.name, sched)


def test_capacity_sweep_small_block(catalogue):
    """Capacities at the start and the end of the output and between, over a block with a long match behind the budget's
    last place (the GPU test takes every capacity)."""
    d = next(c for c in catalogue if c.name == "search-budget-repeat-delta4").data
    r, _ = oracle.encode_hc(d)
    for cap in sorted(set(range(0, 20)) | set(range(r - 20, r + 3)) | set(range(20, r - 20, 97))):
        want = oracle.encode_hc(d, cap=cap)
        assert emu.encode_hc(d, cap=cap) == want, cap
        for smem in (True, False):
            assert emu.encode_hcw(d, cap=cap, smem=smem) == want, (cap, smem)
