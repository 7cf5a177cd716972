"""The measure pass (lz4_measure.cuh) and the packed decode built on it.

CPU: the kernel header runs on the warp emulator and must give the oracle decoders' verdicts -- non-negative results
equal, negative ones by sign.  GPU (H100): lz4b200_measure_batch equals lz4b200_decode_batch's out_len, and
lz4b200_decode_batch_packed lays the decoded blocks back to back without writing anywhere else."""
import hashlib

import numpy as np
import pytest

import oracle
from tests import cases, emu


def _agree(got, want, what=""):
    assert (got < 0) == (want < 0), (what, got, want)
    if want >= 0:
        assert got == want, (what, got, want)


def _expect(c, cap, known):
    return (oracle.decode_known if known else oracle.decode_unknown)(c, cap)[0]


def _corpus(lens=(0, 1, 12, 13, 300, 65536, 65546, 200000)):
    """(compressed, raw) pairs: the oracle's fast and HC output of every content model."""
    out = []
    for i, m in enumerate(cases.MODELS):
        for n in lens:
            d = cases.content(m, n, seed=80 + i).tobytes()
            for fn in (oracle.encode, oracle.encode_hc):
                out.append((fn(d)[1], d))
    return out


def _corrupt(count=400):
    rng = np.random.default_rng(5)
    comp, caps = [], []
    for i in range(count):
        d = cases.content("mixed", 2500, seed=i).tobytes()
        c = bytearray(oracle.encode(d)[1])
        kind = i % 3
        if kind == 0:
            for _ in range(int(rng.integers(1, 4))):
                c[int(rng.integers(0, len(c)))] ^= 1 << int(rng.integers(0, 8))
        elif kind == 1:
            c = c[: int(rng.integers(1, len(c)))]
        else:
            c[int(rng.integers(0, len(c)))] = 0xFF
        comp.append(bytes(c)); caps.append(len(d))
    return comp, caps


def _size_cases():
    """original/fuzzer.c:176-210: exact size, size +-1, one byte short / long -- (compressed, cap, known)."""
    from lz4net_b200 import synth
    out = []
    for seed in range(6):
        d = synth.fuz_block(seed, 6000).tobytes()
        c = oracle.encode(d)[1]
        n = len(d)
        for osz in (n, n - 1, n + 1):
            out.append((c, osz, True))
        for cc, osz in ((c, n + 1), (c, n), (c, n - 1), (c[:-1], n), (c + b"\0", n)):
            out.append((cc, osz, False))
    return out


OVERFLOW = bytes([0x0F, 0, 0]) + b"\xff" * (1 << 16)          # original/fuzzer.c:96-116: a match length that never ends
LONG_LITERAL = bytes([0xF0]) + b"\xff" * 5000                   # a literal length that runs into the end of the stream


# ---- CPU: the kernel header on the warp emulator --------------------------------------------------------------------
@pytest.mark.parametrize("known", [True, False])
def test_measure_matches_oracle_decoders(known):
    pairs = _corpus()
    comp = [c for c, _ in pairs]
    caps = [len(d) for _, d in pairs]
    res = emu.measure(comp, caps, known=known, sched_seed=3)
    for (c, d), cap, r in zip(pairs, caps, res):
        _agree(r, _expect(c, cap, known), len(d))
        if r >= 0:
            assert r == (len(c) if known else len(d))
    if not known:                                                # capacity one byte more / less than the decoded size
        for delta in (1, -1):
            caps2 = [max(len(d) + delta, 0) for _, d in pairs]
            for (c, d), cap, r in zip(pairs, caps2, emu.measure(comp, caps2, known=False, sched_seed=4)):
                _agree(r, _expect(c, cap, False), (len(d), cap))


def test_measure_size_invariants():
    sc = _size_cases()
    for known in (True, False):
        sel = [(c, cap) for c, cap, k in sc if k == known]
        res = emu.measure([c for c, _ in sel], [cap for _, cap in sel], known=known, sched_seed=11)
        expect = [_expect(c, cap, known) for c, cap in sel]
        for r, e in zip(res, expect):
            _agree(r, e)
        assert any(e < 0 for e in expect) and any(e >= 0 for e in expect)


@pytest.mark.parametrize("known", [True, False])
def test_measure_corrupt_streams(known):
    comp, caps = _corrupt()
    res = emu.measure(comp, caps, known=known, sched_seed=13)
    expect = [_expect(c, cap, known) for c, cap in zip(comp, caps)]
    for r, e in zip(res, expect):
        _agree(r, e)
    assert sum(e < 0 for e in expect) > 50 and sum(e >= 0 for e in expect) > 20
    # unlimited capacity: the verdicts at INT32_MAX are those at 256 * len + 64 (no stream of len bytes writes more)
    if not known:
        res = emu.measure(comp, None, known=False, sched_seed=15)
        for c, r in zip(comp, res):
            _agree(r, oracle.decode_unknown(c, 256 * len(c) + 64)[0])


def test_measure_length_overflow_inputs():
    for bad in (OVERFLOW, LONG_LITERAL, OVERFLOW[:3], bytes([0xF0])):
        for known in (True, False):
            cap = 1 << 20
            _agree(emu.measure([bad], [cap], known=known)[0], _expect(bad, cap, known), (len(bad), known))
        assert emu.measure([bad], None)[0] < 0


def test_measure_unlimited_capacity():
    pairs = _corpus(lens=(0, 1, 13, 300, 65536, 65546))
    comp = [c for c, _ in pairs]
    res = emu.measure(comp, None, known=False, sched_seed=7)
    for (c, d), r in zip(pairs, res):
        _agree(r, oracle.decode_unknown(c, 256 * len(c) + 64)[0], len(d))
        assert r == len(d)


@pytest.mark.parametrize("skew", [1, 5, 11, 15])
def test_measure_unaligned_streams_and_lane_schedules(skew):
    pairs = _corpus(lens=(13, 300, 4097, 65536))
    comp = [c for c, _ in pairs]
    for seed in (skew, 100 + skew):
        for known in (True, False):
            res = emu.measure(comp, [len(d) for _, d in pairs], known=known, sched_seed=seed, src_skew=skew)
            assert res == [len(c) if known else len(d) for c, d in pairs]


def test_measure_never_reads_past_the_last_unit():
    """The block's 16-byte-aligned end is the end of a mapped page (the next one is PROT_NONE): a read of any unit
    behind the block's last one would fault.  Valid and truncated streams, both modes."""
    for m, n in (("E0", 65536), ("E50", 65536), ("ETEXT", 20000), ("E100", 65536), ("runs", 9000), ("mixed", 13)):
        d = cases.content(m, n, seed=n % 89).tobytes()
        for fn in (oracle.encode, oracle.encode_hc):
            c = fn(d)[1]
            for cc in (c, c[:-1], c[: len(c) // 2], c[:1]):
                for known in (True, False):
                    _agree(emu.measure([cc], [len(d)], known=known, fence="behind")[0], _expect(cc, len(d), known), (m, n, len(cc), known))
                _agree(emu.measure([cc], fence="behind")[0], oracle.decode_unknown(cc, 256 * len(cc) + 64)[0], (m, n, len(cc)))
    for bad in (OVERFLOW, LONG_LITERAL):
        assert emu.measure([bad], fence="behind")[0] < 0 and emu.measure([bad], [1 << 20], known=True, fence="behind")[0] < 0


def test_entry_points_reject_bad_arguments():
    """A NULL context, or NULL capacities with known sizes: LZ4B200_E_ARG from both entry points, with or without a GPU."""
    from lz4net_b200 import build, native
    build.build()
    l = native.lib()
    b = np.zeros(64, np.uint8); off = np.zeros(4, np.int64); ln = np.ones(4, np.int32); out = np.zeros(4, np.int32)
    assert l.lz4b200_measure_batch(None, b.ctypes.data, off.ctypes.data, ln.ctypes.data, ln.ctypes.data, out.ctypes.data, 1, 0,
                                   native.MEM_HOST, None) == native.E_ARG
    assert l.lz4b200_measure_batch(None, b.ctypes.data, off.ctypes.data, ln.ctypes.data, None, out.ctypes.data, 1, 1,
                                   native.MEM_HOST, None) == native.E_ARG
    assert "dst_cap" in native.last_error()
    assert l.lz4b200_decode_batch_packed(None, b.ctypes.data, off.ctypes.data, ln.ctypes.data, b.ctypes.data, 64,
                                         off.ctypes.data, out.ctypes.data, 1, None) == native.E_ARG


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@pytest.fixture(params=[0, 1, 16], ids=["auto", "lpb", "lanes16"])
def lanes(ctx, request):
    if request.param:
        ctx.set_option("decode_lanes", request.param)
    yield request.param
    ctx.set_option("decode_lanes_auto", 1)


def _gpu_corpus():
    pairs, (bad, bad_caps), sc = _corpus(), _corrupt(120), _size_cases()
    comp = [c for c, _ in pairs] + bad + [OVERFLOW, LONG_LITERAL] + [c for c, _, _ in sc]
    caps = [len(d) for _, d in pairs] + bad_caps + [1 << 20, 1 << 20] + [cap for _, cap, _ in sc]
    return comp, caps


def _device(blocks):
    import torch
    from lz4net_b200.codec import _pack
    src, lens, off = _pack(blocks)
    return torch.from_numpy(src.copy()).cuda(), torch.from_numpy(off).cuda(), torch.from_numpy(lens).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("known", [True, False])
def test_gpu_measure_equals_decode(ctx, lanes, known):
    import torch
    from lz4net_b200 import batch
    comp, caps = _gpu_corpus()
    n = len(comp)
    want, _ = ctx.decode_blocks(comp, caps, known=known)
    assert ctx.measure_blocks(comp, caps, known=known) == want                                   # host memory
    src, so, sl = _device(comp)
    dc = torch.tensor(caps, dtype=torch.int32, device="cuda")
    out = torch.full((n,), 12345, dtype=torch.int32, device="cuda")
    batch.measure(ctx, src, so, sl, out, dst_cap=dc, known=known)                                  # device memory
    assert out.cpu().tolist() == want
    # the device decode gives the same results
    do = torch.from_numpy(np.cumsum(caps) - np.array(caps)).cuda()
    dst = torch.zeros(int(sum(caps)) + 16, dtype=torch.uint8, device="cuda")
    dres = torch.zeros(n, dtype=torch.int32, device="cuda")
    batch.decode(ctx, src, so, sl, dst, do, dc, dres, known=known)
    assert dres.cpu().tolist() == want
    for c, cap, r in zip(comp, caps, want):
        _agree(r, _expect(c, cap, known))


@pytest.mark.gpu
def test_gpu_measure_unlimited_capacity(ctx):
    import torch
    from lz4net_b200 import batch
    comp, _ = _gpu_corpus()
    n = len(comp)
    host = ctx.measure_blocks(comp, None)
    src, so, sl = _device(comp)
    out = torch.zeros(n, dtype=torch.int32, device="cuda")
    batch.measure(ctx, src, so, sl, out)
    assert out.cpu().tolist() == host
    # the decoder at INT32_MAX (a capacity no buffer has: the blocks small enough to give it 256 * len + 64 bytes)
    small = [i for i, c in enumerate(comp) if len(c) <= 4096]
    want, _ = ctx.decode_blocks([comp[i] for i in small], [256 * len(comp[i]) + 64 for i in small], known=False)
    for i, w in zip(small, want):
        _agree(host[i], w)
    for c, r in zip(comp, host):
        _agree(r, oracle.decode_unknown(c, 256 * len(c) + 64)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("cls", ["E0", "E50", "E100", "ETEXT"])
def test_gpu_measure_large_synthetic_batch(ctx, cls):
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 1 << 17, 65536
    slot = oracle.bound(bs)
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID[cls], seed=9)
    so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
    slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.encode(ctx, raw, so, sl, slots, do, dc, clen)
    del raw
    size = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.measure(ctx, slots, do, clen, size)
    assert bool((size == bs).all())
    batch.measure(ctx, slots, do, clen, size, dst_cap=sl, known=True)
    assert torch.equal(size, clen)


def _guarded(t, lo, hi):
    return bool((t[:lo] == 0xA5).all()) and bool((t[hi:] == 0xA5).all())


@pytest.mark.gpu
def test_gpu_decode_packed(ctx, lanes):
    import torch
    from lz4net_b200 import batch
    rng = np.random.default_rng(17)
    blocks, raws = [], []
    for i in range(300):
        m = cases.MODELS[i % len(cases.MODELS)]
        n = int(rng.choice([0, 1, 13, int(rng.integers(14, 5000)), 65536, int(rng.integers(5000, 70000))]))
        d = cases.content(m, n, seed=i).tobytes()
        c = (oracle.encode_hc if i % 3 == 0 else oracle.encode)(d)[1]
        if i % 17 == 5:
            c = c[: len(c) // 2] if len(c) > 2 else b""                                          # truncated
        elif i % 17 == 9:
            c = OVERFLOW
        elif i % 29 == 3:
            c = b""                                                                               # empty block
        blocks.append(c); raws.append(d)
    blocks += _corrupt(60)[0]
    raws += [None] * 60
    n = len(blocks)
    want = [oracle.decode_unknown(c, 256 * len(c) + 64) for c in blocks]
    sizes = [max(r, 0) for r, _ in want]
    need = int(sum(sizes))
    src, so, sl = _device(blocks)
    pad = 4096
    dst = torch.full((need + pad,), 0xA5, dtype=torch.uint8, device="cuda")
    out_off = torch.full((n + 1,), -7, dtype=torch.int64, device="cuda")
    out_len = torch.zeros(n, dtype=torch.int32, device="cuda")
    # too small by one byte: dst untouched, out_len = the sizes, out_off[n] = the need
    view = dst[: need - 1]
    batch.decode_packed(ctx, src, so, sl, view, out_off, out_len)
    torch.cuda.synchronize()
    assert _guarded(dst, 0, 0)
    measured = out_len.cpu().tolist()
    for r, (e, _) in zip(measured, want):
        _agree(r, e)
    assert int(out_off[n]) == need
    # fits exactly (the destination is the first `need` bytes of the guard-filled buffer)
    batch.decode_packed(ctx, src, so, sl, dst[:need], out_off, out_len)
    torch.cuda.synchronize()
    off = out_off.cpu().numpy(); res = out_len.cpu().tolist(); h = dst.cpu().numpy()
    assert off[0] == 0 and list(np.diff(off)) == [max(r, 0) for r in measured]
    assert (h[need:] == 0xA5).all(), "bytes at or past out_off[n] changed"
    for i, ((e, eo), r) in enumerate(zip(want, res)):
        _agree(r, e, i)
        if e >= 0:
            assert h[off[i]:off[i + 1]].tobytes() == eo, i
        else:
            assert off[i + 1] == off[i]
    assert sum(e < 0 for e, _ in want) > 30 and blocks.count(b"") > 3
    # n = 0
    z = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    batch.decode_packed(ctx, src, so[:0], sl[:0], dst, z, out_len[:0])
    torch.cuda.synchronize()
    assert int(z[0]) == 0


@pytest.mark.gpu
def test_gpu_decode_packed_is_asynchronous(ctx):
    """Issued on a non-default stream behind a long kernel: the call returns before its results exist, and the first host
    read after stream.synchronize() sees them."""
    import time
    import torch
    from lz4net_b200 import batch
    blocks = [oracle.encode(cases.content("ETEXT", 65536, seed=i).tobytes())[1] for i in range(64)]
    src, so, sl = _device(blocks)
    dst = torch.empty(64 * 65536, dtype=torch.uint8, device="cuda")
    out_off = torch.full((65,), -1, dtype=torch.int64, device="cuda")
    out_len = torch.full((64,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a = torch.randn(4096, 4096, device="cuda")
        for _ in range(40):
            a = a @ a
            a = a / a.norm()
        t0 = time.perf_counter()
        batch.decode_packed(ctx, src, so, sl, dst, out_off, out_len)
        enqueue = time.perf_counter() - t0
        ev = torch.cuda.Event(); ev.record(s)
    assert not ev.query(), "the packed decode waited for the stream"
    s.synchronize()
    assert out_len.cpu().tolist() == [65536] * 64 and int(out_off[64]) == 64 * 65536
    assert enqueue < 0.5


@pytest.mark.gpu
def test_gpu_decode_packed_large_batch_equals_known_size_decode(ctx):
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 1 << 18, 65536
    slot = oracle.bound(bs)
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID["E50"], seed=21)
    so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
    slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.encode(ctx, raw, so, sl, slots, do, dc, clen)
    del raw
    out = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    res = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.decode(ctx, slots, do, clen, out, so, sl, res, known=True)
    torch.cuda.synchronize()
    assert torch.equal(res, clen)
    h_known = hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()
    out.fill_(0)
    out_off = torch.zeros(nb + 1, dtype=torch.int64, device="cuda")
    batch.decode_packed(ctx, slots, do, clen, out, out_off, res)
    torch.cuda.synchronize()
    assert bool((res == bs).all()) and int(out_off[nb]) == nb * bs
    assert hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest() == h_known
