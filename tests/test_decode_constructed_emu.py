"""CPU: the constructed streams of tests/lz4seq.py through every decoder kernel on the warp emulator.

Each case puts one byte on an accept / reject rule of the reference decoders or on an internal threshold of a kernel
(the group fast path's 32 / 64 / DEC_AHEAD / cap - 112, the TMA chunk and ring boundaries, the lpb output window and
input rings).  Every configuration -- the group decoders at 32 / 16 / 8 / 4 lanes, their output-staged variants, the
lane-per-block decoder in the kernel's geometry and in the emulator's larger one -- must return what the oracle port
returns (tests/test_oracle.py pins the port to the reference on this corpus), known and unknown size: the same verdict,
the same non-negative result and the same bytes, with nothing written outside the destination slot.  The measure pass
must give the same results, and no decoder may read a 16-byte unit that holds no stream byte."""
import functools

import pytest

import oracle
from tests import emu, lz4seq
from tests.test_oracle import CONSTRUCTED_SEED

# emu.decode's lanes: the group decoders (G), their output-staged variants (100 + G), the lane-per-block decoder (1: the
# kernel's geometry LpbGeom<128, 256, 32, 0, 2>; 2: LpbGeom<256, 512, 64, 1, 1>)
CONFIGS = (32, 16, 8, 4, 132, 116, 108, 104, 1, 2)


@functools.lru_cache(maxsize=None)
def _corpus():
    return lz4seq.corpus(CONSTRUCTED_SEED)


@functools.lru_cache(maxsize=None)
def _expected(known):
    fn = oracle.decode_known if known else oracle.decode_unknown
    return [fn(c.stream, c.cap) for c in _corpus()]


def _check(cases, expected, res, outs, known, who):
    for c, (er, eo), r, o in zip(cases, expected, res, outs):
        assert (r < 0) == (er < 0), (who, c.name, r, er)
        if er >= 0:
            assert r == er, (who, c.name, r, er)
            assert (o if known else o[:r]) == eo, (who, c.name, "bytes differ")


@pytest.mark.parametrize("known", [True, False], ids=["known", "unknown"])
@pytest.mark.parametrize("lanes", CONFIGS)
def test_every_decoder_equals_the_oracle(lanes, known):
    """The whole corpus in one batch, then its small blocks again under another lane schedule and other alignments of
    the stream and the destination (emu.decode checks the destination's red zones on every call)."""
    cases, exp = _corpus(), _expected(known)
    blocks, caps = [c.stream for c in cases], [c.cap for c in cases]
    res, outs = emu.decode(blocks, caps, lanes=lanes, known=known, sched_seed=lanes, src_skew=lanes % 16,
                           dst_skew=(3 * lanes) % 16)
    _check(cases, exp, res, outs, known, lanes)
    small = [i for i, c in enumerate(cases) if len(c.stream) <= 2048]
    res, outs = emu.decode([blocks[i] for i in small], [caps[i] for i in small], lanes=lanes, known=known,
                           sched_seed=1000 + lanes, src_skew=(7 * lanes + 5) % 16, dst_skew=(lanes + 9) % 16)
    _check([cases[i] for i in small], [exp[i] for i in small], res, outs, known, (lanes, "second schedule"))


@pytest.mark.parametrize("known", [True, False], ids=["known", "unknown"])
def test_measure_equals_the_decoders(known):
    """lz4_measure.cuh on the same corpus: a non-negative result equals the decoders', a negative one agrees in sign."""
    cases, exp = _corpus(), _expected(known)
    blocks, caps = [c.stream for c in cases], [c.cap for c in cases]
    for seed, skew in ((1, 0), (7, 11)):
        for c, (er, _), r in zip(cases, exp, emu.measure(blocks, caps, known=known, sched_seed=seed, src_skew=skew)):
            assert (r < 0) == (er < 0) and (er < 0 or r == er), (c.name, r, er)


def _fence_cases():
    """Blocks whose last (or first) unit the decoders reach on their careful / general paths: the tail rules, the
    near-end offsets and ring windows, truncated and extended streams, and a placement case per chunk size."""
    pick = []
    for c in _corpus():
        n = c.name
        if ((n.startswith("tail/L5/") and "/cap+0" in n and ("/t4/" in n or "/t5/" in n or "/t12/" in n)) or
                ("/near/" in n and ("/M13/" in n or "/M64/" in n) and "/off" in n and ("/r1/" in n or "/L7/" in n)) or
                "/cut" in n or "/append" in n or (n.startswith("place/") and "/j1/back0/k3/" in n)):
            pick.append(c)
    return pick[::3]


@pytest.mark.parametrize("fence", ["behind", "front"])
def test_decoders_read_only_the_units_that_hold_stream_bytes(fence):
    """Each block lies 0-3 bytes from a PROT_NONE page, behind its last byte or in front of its first: a read of any
    16-byte unit outside [src, src + isize) rounded out to 16 bytes kills the process."""
    cases = _fence_cases()
    assert len(cases) > 40
    for i, c in enumerate(cases):
        for known in (True, False):
            er, eo = (oracle.decode_known if known else oracle.decode_unknown)(c.stream, c.cap)
            for lanes in CONFIGS:
                pad = (i + lanes) % 4
                res, outs = emu.decode([c.stream], [c.cap], lanes=lanes, known=known, fence=fence, pad=pad, sched_seed=i + 1)
                _check([c], [(er, eo)], res, outs, known, (lanes, fence, pad))


def test_careful_paths_reject_at_the_same_byte():
    """The end-of-block cases (lz4seq's tail family): the sequence that decides is always on the group decoders' careful
    path, the lpb decoder's general code and the measure pass, which restate the same rules one by one -- so a rejected
    block gets the same negative result (-(stream position) - 1) from every one of them.  (lz4net sees only the sign; a
    rule moved to a byte where it still rejects, but later or earlier than the others, shows here and nowhere else.)"""
    cases = [c for c in _corpus() if c.name.startswith("tail/")]
    blocks, caps = [c.stream for c in cases], [c.cap for c in cases]
    for known in (True, False):
        runs = {lanes: emu.decode(blocks, caps, lanes=lanes, known=known, sched_seed=3)[0] for lanes in CONFIGS}
        runs["measure"] = emu.measure(blocks, caps, known=known)
        rejected = 0
        for i, c in enumerate(cases):
            got = {who: r[i] for who, r in runs.items()}
            if got["measure"] < 0:
                rejected += 1
                assert len(set(got.values())) == 1, (c.name, known, got)
        assert rejected > 500
