"""GPU (H100): the constructed streams of tests/lz4seq.py through every decoder kernel, the measure pass and the packed
decode, compared with the oracle port (which tests/test_oracle.py pins to the reference on this corpus).

What the emulator cannot vouch for is exercised here: the TMA ring and its mbarrier phases, the real cp.async ordering
of the lane-per-block decoder, and persistent warps that take blocks of very different cost from one counter.  Device
memory slots sit between sentinel-filled gaps, which must be intact after every call."""
import functools

import numpy as np
import pytest

import oracle
from tests import lz4seq
from tests.test_oracle import CONSTRUCTED_SEED

pytestmark = pytest.mark.gpu

# decode_lanes settings: the group decoders, their output-staged variants (100 + G), the lane-per-block decoder (1);
# 0 = the library's own choice
LANES = (32, 16, 8, 4, 132, 116, 108, 104, 1, 0)
SENTINEL = 0xA5


@functools.lru_cache(maxsize=None)
def _corpus():
    return lz4seq.corpus(CONSTRUCTED_SEED)


@functools.lru_cache(maxsize=None)
def _expected(known):
    fn = oracle.decode_known if known else oracle.decode_unknown
    return [fn(c.stream, c.cap) for c in _corpus()]


@functools.lru_cache(maxsize=None)
def _unlimited():
    """Unknown-size results at a capacity no block of the corpus reaches (the measure pass's INT32_MAX)."""
    return [oracle.decode_unknown(c.stream, 256 * len(c.stream) + 64) for c in _corpus()]


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@pytest.fixture(params=LANES, ids=lambda v: f"lanes{v}" if v else "auto")
def lanes(ctx, request):
    if request.param:
        ctx.set_option("decode_lanes", request.param)
    else:
        ctx.set_option("decode_lanes_auto", 1)
    yield request.param
    ctx.set_option("decode_lanes_auto", 1)


def _agree(got, want, what):
    assert (got < 0) == (want < 0), (what, got, want)
    if want >= 0:
        assert got == want, (what, got, want)


def _check(cases, expected, res, outs, known, who):
    for c, (er, eo), r, o in zip(cases, expected, res, outs):
        _agree(r, er, (who, c.name))
        if er >= 0:
            assert (o if known else o[:r]) == eo, (who, c.name, "bytes differ")


@pytest.mark.parametrize("known", [True, False], ids=["known", "unknown"])
def test_host_batch_every_decoder(ctx, lanes, known):
    """Host memory (ctx.decode_blocks).  A host batch refuses a negative capacity as an argument error: the one such
    case is left to the device-memory tests."""
    keep = [i for i, c in enumerate(_corpus()) if c.cap >= 0]
    cases = [_corpus()[i] for i in keep]
    res, outs = ctx.decode_blocks([c.stream for c in cases], [c.cap for c in cases], known=known)
    _check(cases, [_expected(known)[i] for i in keep], res, outs, known, lanes)


def _layout(sizes, gap, rng):
    """Offsets of slots of these sizes, each behind a gap of gap + 0..15 bytes (every alignment); returns (offsets, total)."""
    off, p = [], 0
    for s in sizes:
        p += gap + int(rng.integers(0, 16))
        off.append(p)
        p += max(int(s), 0)
    return np.array(off, np.int64), p + gap


def _device_batch(cases, rng):
    """The streams in device memory (random alignments, sentinel gaps) and destination slots of cap bytes each between
    sentinel-filled gaps.  Returns tensors (src, so, sl, dst, do, dc) and the host layout of dst (offsets, total)."""
    import torch
    so, stotal = _layout([len(c.stream) for c in cases], 16, rng)
    src = np.full(stotal, SENTINEL, np.uint8)
    for o, c in zip(so, cases):
        src[o:o + len(c.stream)] = np.frombuffer(c.stream, np.uint8)
    caps = np.array([c.cap for c in cases], np.int32)
    do, dtotal = _layout(caps, 64, rng)
    dev = lambda a: torch.from_numpy(a).cuda()
    dst = torch.full((dtotal,), SENTINEL, dtype=torch.uint8, device="cuda")
    sl = np.array([len(c.stream) for c in cases], np.int32)
    return (dev(src), dev(so), dev(sl), dst, dev(do), dev(caps)), do


def _check_device(cases, expected, res, dst, do, known, who):
    """Results and bytes as the oracle's; every byte outside the slots [do[i], do[i] + cap) still the sentinel."""
    h = dst.cpu().numpy()
    inside = np.zeros(h.size, bool)
    outs = []
    for c, o in zip(cases, do):
        inside[o:o + max(c.cap, 0)] = True
        outs.append(h[o:o + max(c.cap, 0)].tobytes())
    assert (h[~inside] == SENTINEL).all(), (who, "a decoder wrote outside its slot")
    _check(cases, expected, res, outs, known, who)


@pytest.mark.parametrize("known", [True, False], ids=["known", "unknown"])
def test_device_batch_every_decoder_keeps_the_gaps(ctx, lanes, known):
    import torch
    from lz4net_b200 import batch
    cases = _corpus()
    (src, so, sl, dst, do_t, dc), do = _device_batch(cases, np.random.default_rng(lanes + 10 * known))
    res = torch.full((len(cases),), 12345, dtype=torch.int32, device="cuda")
    batch.decode(ctx, src, so, sl, dst, do_t, dc, res, known=known)
    torch.cuda.synchronize()
    _check_device(cases, _expected(known), res.cpu().tolist(), dst, do, known, lanes)


@pytest.mark.parametrize("known", [True, False], ids=["known", "unknown"])
def test_device_measure(ctx, known):
    import torch
    from lz4net_b200 import batch
    cases = _corpus()
    (src, so, sl, _, _, dc), _ = _device_batch(cases, np.random.default_rng(3))
    out = torch.full((len(cases),), 12345, dtype=torch.int32, device="cuda")
    batch.measure(ctx, src, so, sl, out, dst_cap=dc, known=known)
    for c, (er, _), r in zip(cases, _expected(known), out.cpu().tolist()):
        _agree(r, er, c.name)
    if not known:
        batch.measure(ctx, src, so, sl, out)                                  # no capacities: INT32_MAX per block
        for c, (er, _), r in zip(cases, _unlimited(), out.cpu().tolist()):
            _agree(r, er, (c.name, "unlimited"))


def test_device_packed_unknown_size_decode(ctx):
    """lz4b200_decode_batch_packed: out_off is the exclusive scan of the oracle's sizes (0 for a rejected block), the
    bytes are the oracle's, and nothing at or behind out_off[n] changes."""
    import torch
    from lz4net_b200 import batch
    cases = _corpus()
    want = _unlimited()
    sizes = [max(r, 0) for r, _ in want]
    need = int(sum(sizes))
    (src, so, sl, _, _, _), _ = _device_batch(cases, np.random.default_rng(4))
    dst = torch.full((need + 4096,), SENTINEL, dtype=torch.uint8, device="cuda")
    n = len(cases)
    out_off = torch.full((n + 1,), -7, dtype=torch.int64, device="cuda")
    out_len = torch.zeros(n, dtype=torch.int32, device="cuda")
    batch.decode_packed(ctx, src, so, sl, dst[:need], out_off, out_len)
    torch.cuda.synchronize()
    off, res, h = out_off.cpu().numpy(), out_len.cpu().tolist(), dst.cpu().numpy()
    assert off.tolist() == [0] + np.cumsum(sizes).tolist()
    assert (h[need:] == SENTINEL).all(), "bytes at or past out_off[n] changed"
    for i, (c, (er, eo), r) in enumerate(zip(cases, want, res)):
        _agree(r, er, c.name)
        if er >= 0:
            assert h[off[i]:off[i + 1]].tobytes() == eo, c.name


@pytest.mark.parametrize("lanes", [0, 1, 4, 104, 32], ids=["auto", "lanes1", "lanes4", "lanes104", "lanes32"])
def test_large_batch_of_mixed_cost(ctx, lanes):
    """The corpus five times over (about 24 000 blocks of 2 bytes to 200 KiB, shuffled): persistent warps and lanes take
    blocks of very different cost from one counter, both sizes, every slot between sentinel gaps."""
    import torch
    from lz4net_b200 import batch
    base = _corpus()
    rng = np.random.default_rng(lanes + 77)
    order = rng.permutation(np.tile(np.arange(len(base)), 5))
    cases = [base[i] for i in order]
    assert len(cases) >= 20_000
    if lanes:
        ctx.set_option("decode_lanes", lanes)
    try:
        for known in (True, False):
            exp = _expected(known)
            (src, so, sl, dst, do_t, dc), do = _device_batch(cases, rng)
            res = torch.full((len(cases),), 12345, dtype=torch.int32, device="cuda")
            batch.decode(ctx, src, so, sl, dst, do_t, dc, res, known=known)
            torch.cuda.synchronize()
            _check_device(cases, [exp[i] for i in order], res.cpu().tolist(), dst, do, known, (lanes, known))
    finally:
        ctx.set_option("decode_lanes_auto", 1)
