"""The fast encoder's rounds (lz4_encode.cuh, find_round) on constructed blocks: CPU warp emulator against the oracle.

A round evaluates 32 or 64 serial iterations of the reference's find-match loop at once.  Where an earlier iteration
of the same round has the same hash, the kernel has to work out the candidate the serial loop would have seen: on the
pair path (two sharers, resolved through the table), the exact path (three or more, or variant 1) or in the fused
round's lanes 0 and 1 and the post-match probe tried alone.  Content rarely reaches the corners of that, so the blocks
here are noise with words planted at chosen iterations of chosen rounds (tests/encround.py), each checked through a
model of the kernel's rounds before any byte is compared.  The model itself is pinned to the kernel through its event
counters (enc_prof.cuh)."""
import pytest

import oracle
from tests import cases, emu, encround

TUNES = [(12, 8, 24), (0, 0, 0), (64, 1000, 1000)]


@pytest.fixture(scope="module")
def catalogue():
    return encround.catalogue()


def test_catalogue_covers_the_round(catalogue):
    """The planted structures the catalogue exists for are all there (each builder has checked its own)."""
    names = [c.name for c in catalogue]
    assert sum(n.startswith("pair-distance-") for n in names) == 31
    assert len(set(names)) == len(names)
    counts = {k: 0 for k in ("pair", "exact")}
    for c in catalogue:
        p = encround.parse(c.data)
        rs, _ = encround.rounds(c.data, p)
        for k in counts:
            counts[k] += any(r.path == k for r in rs)
    assert counts["pair"] >= 60 and counts["exact"] >= 8, counts


@pytest.mark.parametrize("tune", TUNES)
def test_model_counts_equal_the_kernel_counters(catalogue, tune):
    """Rounds (wide, exact, pair) and probes tried alone (hit): the model's counts are the emulated kernel's, for every
    content model and every constructed block, under both variants."""
    blocks = [cases.content(m, n, seed=40 + i).tobytes() for i, m in enumerate(cases.MODELS) for n in (5000, 66000)]
    blocks += [c.data for c in catalogue if len(c.data) < 10000]
    blocks += [c.data for c in catalogue if c.name in ("far-probe-65536", "far-pair-65535", "boundary-65547")]
    for variant in (2, 1):
        for b in blocks:
            r, out, ev = emu.encode_events(b, variant, tune, sched_seed=len(b))
            assert ev == encround.counts(b, variant, tune), (len(b), variant)
            assert (r, out) == oracle.encode(b)


@pytest.mark.parametrize("variant", [2, 1])
@pytest.mark.parametrize("tune", TUNES)
def test_constructed_blocks_match_the_oracle(catalogue, variant, tune):
    k = TUNES.index(tune)
    blocks = [c.data for c in catalogue]
    res, outs = emu.encode(blocks, variant=variant, tune=tune, sched_seed=3 + 5 * k + variant, src_skew=(k + variant) % 4,
                           dst_skew=(3 * k + variant) % 7)
    for c, r, o in zip(catalogue, res, outs):
        assert (r, o) == oracle.encode(c.data), c.name


def test_output_limit_over_a_pair_and_an_exact_case(catalogue):
    """Every capacity from 0 to past the compressed size, over a 600-byte block with a pair hit and one with a hit on
    the exact path."""
    by = {c.name: c.data for c in catalogue}
    for name in ("pair-distance-7", "exact-ABB-r0"):
        b = by[name]
        r, _ = oracle.encode(b)
        caps = list(range(0, r + 3))
        res, outs = emu.encode([b] * len(caps), caps, sched_seed=7)
        for cap, rr, o in zip(caps, res, outs):
            assert (rr, o) == oracle.encode(b, cap=cap), (name, cap)
