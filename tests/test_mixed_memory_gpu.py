"""Mixed-memory batches on an H100: device source -> host destination (lz4b200_encode_batch / decode_batch with
LZ4B200_MEM_DEVICE_TO_HOST, lz4b200_encode_batch_packed_from_device) and host source -> device destination
(LZ4B200_MEM_HOST_TO_DEVICE).

Results and bytes must be those of MEM_DEVICE (and the oracle); a host destination receives only the bytes each block
produced and a device destination is written only inside each block's slot; the call's device accesses are ordered behind
the work already queued on the caller's stream; the wrong kind of memory on either side is refused."""
import functools

import numpy as np
import pytest

import oracle
from tests import cases
from tests.test_measure import _corrupt, _size_cases

pytestmark = pytest.mark.gpu

LENS = (0, 1, 13, 3000, 65536, 65546, 1 << 20)
HOST_GUARD, DEV_GUARD = 0xEE, 0xA5
E_ARG = -1
CHUNK_MB_DEFAULT = 128


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


def _layout(sizes, skew, gap):
    """int64 offsets of `sizes` laid out with `gap` bytes between them, the first `skew` bytes in (misaligned)."""
    sizes = np.maximum(np.asarray(sizes, np.int64), 0)
    off = np.concatenate([[0], np.cumsum(sizes + gap)[:-1]]).astype(np.int64) + skew
    return off, int(off[-1] + sizes[-1] + gap) if len(sizes) else skew + gap


def _src(blocks, skew=3, gap=5):
    so, total = _layout([len(b) for b in blocks], skew, gap)
    buf = np.zeros(total + 16, np.uint8)
    for o, b in zip(so, blocks):
        buf[o:o + len(b)] = np.frombuffer(b, np.uint8)
    return buf, so, np.array([len(b) for b in blocks], np.int32)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(nbytes, fill, pinned):
    """A host uint8 array of nbytes filled with `fill`: plain numpy (pageable) or the numpy view of a pinned torch tensor."""
    import torch
    if pinned:
        return torch.full((nbytes,), fill, dtype=torch.uint8).pin_memory().numpy()
    return np.full(nbytes, fill, np.uint8)


class _Options:
    """Sets context options for a with-block and restores the library defaults afterwards."""
    RESTORE = {"hc_kernel": ("hc_kernel", -1), "host_chunk_mb": ("host_chunk_mb", CHUNK_MB_DEFAULT),
               "decode_lanes": ("decode_lanes_auto", 1)}

    def __init__(self, ctx, **kw):
        self.ctx, self.kw = ctx, kw

    def __enter__(self):
        for k, v in self.kw.items():
            self.ctx.set_option(k, v)

    def __exit__(self, *a):
        for k in self.kw:
            self.ctx.set_option(*self.RESTORE[k])


@functools.lru_cache(maxsize=None)
def _oracle_enc(data, cap, hc):
    return (oracle.encode_hc if hc else oracle.encode)(data, cap=cap)


def _inputs():
    return [cases.content(m, n, seed=60 + i).tobytes() for i, m in enumerate(cases.MODELS) for n in LENS]


def _device_encode(ctx, blocks, caps, hc):
    """MEM_DEVICE encode of the same blocks (same misaligned source layout): (out_len, bytes per block)."""
    import torch
    from lz4net_b200 import batch
    buf, so, sl = _src(blocks)
    do, total = _layout(caps, 0, 0)
    slots = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    out = torch.zeros(len(blocks), dtype=torch.int32, device="cuda")
    batch.encode(ctx, _dev(buf), _dev(so), _dev(sl), slots, _dev(do), _dev(np.asarray(caps, np.int32)), out, hc=hc)
    torch.cuda.synchronize()
    res, h = out.cpu().tolist(), slots.cpu().numpy()
    return res, [h[o:o + max(r, 0)].tobytes() for o, r in zip(do, res)]


def _caps(ctx, blocks, hc):
    """Per block: the bound, the input length, exactly the compressed size, and one byte short of it, in turn."""
    res, _ = _device_encode(ctx, blocks, [oracle.bound(len(b)) for b in blocks], hc)
    return np.array([[oracle.bound(len(b)), len(b), r, max(r - 1, 0)][i % 4] for i, (b, r) in enumerate(zip(blocks, res))], np.int32)


# ---- device -> host encode --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk_mb", [1, CHUNK_MB_DEFAULT], ids=["chunks-of-few-blocks", "one-large-chunk"])
@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("mode", ["fast", "hc-auto", "hc0", "hc1", "hc2"])
def test_gpu_encode_to_host_equals_device_and_oracle(ctx, mode, pinned, chunk_mb):
    """Every content model at lengths 0 .. 1 MiB, misaligned device source, host slots with guard bytes around and
    between them.  With 1 MiB pipeline stages every chunk holds at most eight blocks (one copy per block lands them);
    with the default stage the whole batch is one chunk (compacted on the device, one copy, scattered on the host)."""
    from lz4net_b200 import batch
    hc = mode != "fast"
    blocks = _inputs()
    n = len(blocks)
    with _Options(ctx, **({"hc_kernel": int(mode[2])} if mode.startswith("hc") and mode != "hc-auto" else {})):
        caps = _caps(ctx, blocks, hc)
        want_res, want_out = _device_encode(ctx, blocks, caps, hc)
        buf, so, sl = _src(blocks)
        do, total = _layout(caps, 7, 9)
        dst = _host(total + 64, HOST_GUARD, pinned)
        out = np.full(n, 12345, np.int32)
        raw = _dev(buf)
        with _Options(ctx, host_chunk_mb=chunk_mb):
            batch.encode_to_host(ctx, raw, so, sl, dst, do, caps, out, hc=hc)
    res = out.tolist()
    assert res == want_res
    for i, (b, c, o, r) in enumerate(zip(blocks, caps, do, res)):
        assert dst[o:o + max(r, 0)].tobytes() == want_out[i], (mode, i, len(b), int(c))
        if not hc or len(b) <= 65546 or i % 3 == 0:                                        # (the oracle's HC on 1 MiB is slow)
            assert (r, dst[o:o + max(r, 0)].tobytes()) == _oracle_enc(b, int(c), hc), (mode, i, len(b), int(c))
    written = np.zeros(len(dst), bool)
    for o, r in zip(do, res):
        written[o:o + max(r, 0)] = True
    assert (dst[~written] == HOST_GUARD).all(), "a host byte outside what a block produced changed"
    assert any(r == 0 for r in res) and sum(r > 0 for r in res) > n // 2                 # some blocks did not fit, most did


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("hc", [False, True])
def test_gpu_encode_to_host_packed_equals_host_packed(ctx, hc, pinned):
    """The packed form equals lz4b200_encode_batch_packed on the same data (over many pipeline chunks); one byte short of
    the total is LZ4B200_E_ARG; n = 0 writes out_off[0] = 0."""
    from lz4net_b200 import batch, native
    blocks = _inputs()
    n = len(blocks)
    caps = _caps(ctx, blocks, hc)
    with _Options(ctx, host_chunk_mb=1):
        want_res, want_off, want_packed = ctx.encode_blocks_packed(blocks, caps=caps, hc=hc)
        buf, so, sl = _src(blocks)
        raw = _dev(buf)
        total = want_off[-1]
        dst = _host(total + 64, HOST_GUARD, pinned)
        out = np.zeros(n, np.int32)
        off = np.full(n + 1, -7, np.int64)
        assert batch.encode_to_host_packed(ctx, raw, so, sl, caps, dst[:total], off, out, hc=hc) == total
        assert out.tolist() == want_res and off.tolist() == want_off
        assert dst[:total].tobytes() == want_packed and (dst[total:] == HOST_GUARD).all()
        short = _host(total - 1, HOST_GUARD, pinned)
        rc = native.lib().lz4b200_encode_batch_packed_from_device(
            ctx.handle, raw.data_ptr(), so.ctypes.data, sl.ctypes.data, caps.ctypes.data, short.ctypes.data, total - 1,
            off.ctypes.data, out.ctypes.data, n, int(hc), 0)
        assert rc == E_ARG
    z = np.full(1, -7, np.int64)
    e64, e32 = np.zeros(0, np.int64), np.zeros(0, np.int32)
    assert batch.encode_to_host_packed(ctx, raw, e64, e32, e32, np.zeros(16, np.uint8), z, e32, hc=hc) == 0 and z[0] == 0


# ---- host -> device decode --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _decode_corpus(known):
    """(compressed, capacity): the oracle's fast output of every content model and its HC output up to 65 546 bytes, the
    corruption cases of the measure tests, and the exact / one-short / one-long capacities of the fuzzer's size cases."""
    comp, caps = [], []
    for i, m in enumerate(cases.MODELS):
        for n in LENS:
            d = cases.content(m, n, seed=80 + i).tobytes()
            for fn in (oracle.encode, oracle.encode_hc) if n <= 65546 else (oracle.encode,):
                comp.append(fn(d)[1]); caps.append(n)
    bad, bad_caps = _corrupt(120)
    comp += bad; caps += bad_caps
    for c, cap, k in _size_cases():
        if k == known:
            comp.append(c); caps.append(cap)
    return comp, np.array(caps, np.int32)


def _device_decode(ctx, comp, caps, known):
    """MEM_DEVICE decode of the same blocks into guarded slots: (out_len, device slot bytes as a host array, dst_off)."""
    import torch
    from lz4net_b200 import batch
    buf, so, sl = _src(comp, skew=5, gap=3)
    do, total = _layout(caps, 11, 13)
    out_t = torch.full((total + 64,), DEV_GUARD, dtype=torch.uint8, device="cuda")
    res = torch.full((len(comp),), 12345, dtype=torch.int32, device="cuda")
    batch.decode(ctx, _dev(buf), _dev(so), _dev(sl), out_t, _dev(do), _dev(caps), res, known=known)
    torch.cuda.synchronize()
    return res.cpu().tolist(), out_t.cpu().numpy(), do


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("lanes", [0, 16, 1], ids=["auto", "lanes16", "lpb"])
@pytest.mark.parametrize("known", [True, False], ids=["known", "unknown"])
def test_gpu_decode_from_host_equals_device(ctx, known, lanes, pinned):
    """Statuses and decoded bytes equal MEM_DEVICE's (exactly with a pinned decoder; with the auto-picked one, which may
    pick a different decoder per pipeline chunk, non-negative results exactly and negative ones by sign), over many
    pipeline chunks; no device byte outside a block's slot changes."""
    import torch
    from lz4net_b200 import batch
    comp, caps = _decode_corpus(known)
    n = len(comp)
    with _Options(ctx, **({"decode_lanes": lanes} if lanes else {})):
        want, want_h, do = _device_decode(ctx, comp, caps, known)
        buf, so, sl = _src(comp, skew=5, gap=3)
        src = _host(len(buf), 0, pinned)
        src[:] = buf
        _, total = _layout(caps, 11, 13)
        out_t = torch.full((total + 64,), DEV_GUARD, dtype=torch.uint8, device="cuda")
        res = np.full(n, 12345, np.int32)
        with _Options(ctx, host_chunk_mb=1):
            batch.decode_from_host(ctx, src, so, sl, out_t, do, caps, res, known=known)
    got, h = res.tolist(), out_t.cpu().numpy()
    for i, (g, w) in enumerate(zip(got, want)):
        if lanes:
            assert g == w, (i, g, w)
        else:
            assert (g < 0) == (w < 0) and (w < 0 or g == w), (i, g, w)
        if w >= 0:
            m = int(caps[i]) if known else w
            assert h[do[i]:do[i] + m].tobytes() == want_h[do[i]:do[i] + m].tobytes(), i
    slot = np.zeros(len(h), bool)
    for o, c in zip(do, caps):
        slot[o:o + max(int(c), 0)] = True
    assert (h[~slot] == DEV_GUARD).all(), "a device byte outside [dst_off, dst_off + dst_cap) changed"
    assert any(g < 0 for g in got) and sum(g >= 0 for g in got) > n // 2


# ---- ordering behind the caller's stream ------------------------------------------------------------------------------
def _busy(s):
    """A few hundred milliseconds of work queued on stream s."""
    import torch
    with torch.cuda.stream(s):
        a = torch.randn(4096, 4096, device="cuda")
        for _ in range(40):
            a = a @ a
            a = a / a.norm()


def test_gpu_encode_to_host_waits_for_the_producer_on_its_stream(ctx):
    """synth_fill queued on a non-default stream behind a long kernel chain, then at once a device -> host encode given that
    stream: the encode reads the filled data, the same as after a synchronise."""
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 512, 65536
    so = np.arange(nb, dtype=np.int64) * bs
    sl = np.full(nb, bs, np.int32)
    caps = np.full(nb, oracle.bound(bs), np.int32)
    do = np.arange(nb, dtype=np.int64) * int(caps[0])

    def run(sync):
        raw = torch.zeros(nb * bs, dtype=torch.uint8, device="cuda")
        dst = np.zeros(nb * int(caps[0]), np.uint8)
        out = np.zeros(nb, np.int32)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        _busy(s)
        with torch.cuda.stream(s):
            batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID["E50"], seed=5)
            if sync:
                s.synchronize()
            batch.encode_to_host(ctx, raw, so, sl, dst, do, caps, out)
        return out, dst

    out0, dst0 = run(False)
    out1, dst1 = run(True)
    assert np.array_equal(out0, out1) and np.array_equal(dst0, dst1)
    assert (out1 > 0).all() and (out1 < bs).all()                                          # E50 data, not zeros


def test_gpu_decode_from_host_waits_for_readers_of_the_old_contents(ctx):
    """A dst.clone() queued on a non-default stream behind a long kernel chain, then at once a host -> device decode into
    dst given that stream: the clone holds the old contents, not the decoded bytes."""
    import torch
    from lz4net_b200 import batch
    blocks = [cases.content("ETEXT", 65536, seed=i).tobytes() for i in range(64)]
    comp = [oracle.encode(b)[1] for b in blocks]
    buf, so, sl = _src(comp)
    caps = np.full(len(blocks), 65536, np.int32)
    do = np.arange(len(blocks), dtype=np.int64) * 65536
    dst = torch.full((len(blocks) * 65536,), 0x5A, dtype=torch.uint8, device="cuda")
    res = np.zeros(len(blocks), np.int32)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    _busy(s)
    with torch.cuda.stream(s):
        snap = dst.clone()
        batch.decode_from_host(ctx, buf, so, sl, dst, do, caps, res)
    s.synchronize()
    assert bool((snap == 0x5A).all()), "the decode overwrote dst before an earlier reader on the stream was done"
    assert res.tolist() == [len(c) for c in comp]
    assert dst.cpu().numpy().tobytes() == b"".join(blocks)


# ---- the wrong kind of memory -----------------------------------------------------------------------------------------
def test_gpu_mixed_calls_refuse_the_wrong_kind_of_memory(ctx):
    import torch
    from lz4net_b200 import native
    l = native.lib()
    n = 4
    so = np.arange(n, dtype=np.int64) * 100
    sl = np.full(n, 100, np.int32)
    cap = np.full(n, oracle.bound(100), np.int32)
    do = np.arange(n, dtype=np.int64) * int(cap[0])
    out = np.zeros(n, np.int32)
    off = np.zeros(n + 1, np.int64)
    h_src, h_dst = np.zeros(n * 100 + 16, np.uint8), np.zeros(n * int(cap[0]) + 16, np.uint8)
    d_src = torch.zeros(n * 100 + 16, dtype=torch.uint8, device="cuda")
    d_dst = torch.zeros(n * int(cap[0]) + 16, dtype=torch.uint8, device="cuda")
    p = lambda a: a.ctypes.data                                                              # noqa: E731

    def enc(src, dst, mem):
        return l.lz4b200_encode_batch(ctx.handle, src, p(so), p(sl), dst, p(do), p(cap), p(out), n, 0, mem, 0)

    def dec(src, dst, mem):
        return l.lz4b200_decode_batch(ctx.handle, src, p(so), p(sl), dst, p(do), p(sl), p(out), n, 1, mem, 0)

    D2H, H2D = native.MEM_DEVICE_TO_HOST, native.MEM_HOST_TO_DEVICE
    assert enc(p(h_src), p(h_dst), D2H) == E_ARG                                           # host src as the device side
    assert enc(d_src.data_ptr(), d_dst.data_ptr(), D2H) == E_ARG                           # device dst as the host side
    assert dec(d_src.data_ptr(), d_dst.data_ptr(), H2D) == E_ARG                           # device src as the host side
    assert dec(p(h_src), p(h_dst), H2D) == E_ARG                                           # host dst as the device side
    assert l.lz4b200_encode_batch_packed_from_device(ctx.handle, p(h_src), p(so), p(sl), p(cap), p(h_dst), len(h_dst),
                                                     p(off), p(out), n, 0, 0) == E_ARG
    for mem in (D2H, H2D):
        assert l.lz4b200_measure_batch(ctx.handle, p(h_src), p(so), p(sl), None, p(out), n, 0, mem, 0) == E_ARG
    assert enc(d_src.data_ptr(), p(h_dst), D2H) == 0 and dec(p(h_src), d_dst.data_ptr(), H2D) == 0     # the right sides


# ---- round trip -------------------------------------------------------------------------------------------------------
def test_gpu_large_e50_round_trip_through_host_memory(ctx):
    """2^14 x 64 KiB E50 blocks: device -> packed host encode -> host -> device known-size decode; equal on the device."""
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 1 << 14, 65536
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID["E50"], seed=21)
    so = np.arange(nb, dtype=np.int64) * bs
    sl = np.full(nb, bs, np.int32)
    caps = np.full(nb, oracle.bound(bs), np.int32)
    packed = np.empty(nb * int(caps[0]), np.uint8)
    off = np.zeros(nb + 1, np.int64)
    clen = np.zeros(nb, np.int32)
    total = batch.encode_to_host_packed(ctx, raw, so, sl, caps, packed, off, clen)
    assert (clen > 0).all() and (clen < bs).all() and total == int(clen.sum())
    out = torch.zeros_like(raw)
    res = np.zeros(nb, np.int32)
    batch.decode_from_host(ctx, packed, off[:-1].copy(), clen, out, so, sl, res)
    assert np.array_equal(res, clen)
    assert torch.equal(out, raw)
