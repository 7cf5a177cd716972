"""The asynchronous packed decode, Wrap and Unwrap calls on an H100: lz4b200_wrap_batch_packed_from_device_async (device
inputs wrapped back to back into page-locked host memory), lz4b200_unwrap_batch_to_device_async and its packed form
(page-locked packets restored into device memory, headers read on the device), and
lz4b200_decode_batch_packed_to_device_async.

Results and bytes must be those of the synchronous calls however many pipeline stages a batch spans; a destination too
small follows the packed calls' contract with nothing written behind its capacity; the Unwraps must read headers that
work queued before them on the stream is still writing; the calls return while the device is busy, are ordered on the
caller's stream, and refuse the wrong kind of memory, negative lengths and a capturing stream."""
import functools
import struct

import numpy as np
import pytest

import oracle
from tests import cases
from tests.test_mixed_memory_gpu import _dev, _layout, _Options, _src
from tests.test_wrap_mixed_gpu import _status_cases

pytestmark = pytest.mark.gpu

CLASSES = ("E0", "E50", "E100", "ETEXT")
SIZES = (0, 1, 13, 65536, 65547, 1 << 20)
CANARY = 0x5C
E_ARG, E_FORMAT = -1, -5


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@functools.lru_cache(maxsize=None)
def _blocks():
    return tuple(cases.content(m, n, seed=60 + i).tobytes() for i, m in enumerate(CLASSES) for n in SIZES)


def _pinned(n, fill, dtype=None):
    import torch
    return torch.full((n,), fill, dtype=dtype or torch.uint8).pin_memory()


def _pinned_bytes(buf):
    t = _pinned(len(buf), 0)
    t.numpy()[:] = buf
    return t


def _outs(n, kind):
    """out_off (int64[n+1]) and out_len (int32[n]) in device memory or page-locked host memory, filled with junk."""
    import torch
    if kind == "device":
        return (torch.full((n + 1,), -7, dtype=torch.int64, device="cuda"), torch.full((n,), 12345, dtype=torch.int32, device="cuda"))
    return _pinned(n + 1, -7, torch.int64), _pinned(n, 12345, torch.int32)


def _sync_wrap(ctx, raw, so, sl, hc):
    from lz4net_b200 import batch
    n = len(so)
    dst = np.zeros(int(sl.sum()) + 8 * n + 64, np.uint8)
    off, res = np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
    total = batch.wrap_to_host_packed(ctx, raw, so, sl, dst, off, res, hc=hc)
    return res, off, dst[:total].tobytes()


def _packets(ctx, hc=False):
    """(packet bytes, the inputs): the synchronous packed Wrap of _blocks(), cut into packets."""
    blocks = _blocks()
    buf, so, sl = _src(blocks)
    res, off, wire = _sync_wrap(ctx, _dev(buf), so, sl, hc)
    return [wire[off[i]:off[i + 1]] for i in range(len(blocks))], blocks


# ---- Wrap -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["device", "pinned"])
@pytest.mark.parametrize("hc", [False, True], ids=["fast", "hc"])
def test_gpu_async_wrap_equals_the_synchronous_packed_wrap(ctx, hc, kind):
    import torch
    from lz4net_b200 import batch
    blocks = _blocks()
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    with _Options(ctx, host_chunk_mb=1):                              # more stages than the two asynchronous slots
        want_res, want_off, want = _sync_wrap(ctx, raw, so, sl, hc)
        total = int(want_off[-1])
        dst = _pinned(total + 256, CANARY)
        off, res = _outs(n, kind)
        batch.wrap_to_host_packed_async(ctx, raw, so, sl, dst, off, res, hc=hc)
        torch.cuda.synchronize()
    assert res.cpu().numpy().tolist() == want_res.tolist()
    assert np.array_equal(off.cpu().numpy(), want_off)
    h = dst.numpy()
    assert h[:total].tobytes() == want and (h[total:] == CANARY).all()
    assert all(r <= len(b) + 8 for r, b in zip(want_res, blocks))       # incompressible inputs are stored raw


def test_gpu_async_wrap_into_a_destination_too_small(ctx):
    import torch
    from lz4net_b200 import batch
    blocks = _blocks()
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    with _Options(ctx, host_chunk_mb=1):
        want_res, want_off, want = _sync_wrap(ctx, raw, so, sl, False)
        total = int(want_off[-1])
        for short in (1, total // 2, total - 1):
            alloc = _pinned(total + 4096, CANARY)
            off, res = _outs(n, "pinned")
            batch.wrap_to_host_packed_async(ctx, raw, so, sl, alloc[:total - short], off, res)
            torch.cuda.synchronize()
            assert res.numpy().tolist() == want_res.tolist() and np.array_equal(off.numpy(), want_off)
            h = alloc.numpy()
            assert (h[total - short:] == CANARY).all(), short             # nothing behind dst_total_cap


# ---- Unwrap into slots ------------------------------------------------------------------------------------------------
def _slots_case(ctx, which):
    """(packets, capacities): round-trip packets with 0-2 spare bytes, or every rejection of the synchronous tests."""
    if which == "round-trip":
        packets, blocks = _packets(ctx, hc=True)
        return packets, [len(d) + i % 3 for i, d in enumerate(blocks)]
    pairs = _status_cases(ctx)
    return [p for p, _ in pairs], [max(c, 0) for _, c in pairs]


@pytest.mark.parametrize("kind", ["device", "pinned"])
@pytest.mark.parametrize("which", ["round-trip", "statuses"])
def test_gpu_async_unwrap_equals_the_synchronous_unwrap_to_device(ctx, which, kind):
    import torch
    from lz4net_b200 import batch
    packets, caps = _slots_case(ctx, which)
    n = len(packets)
    buf, so, sl = _src(packets, skew=5, gap=3)
    caps = np.asarray(caps, np.int32)
    do, total = _layout(caps, 11, 13)
    with _Options(ctx, host_chunk_mb=1):
        want_t = torch.full((total + 64,), CANARY, dtype=torch.uint8, device="cuda")
        want_res = np.full(n, 12345, np.int32)
        batch.unwrap_to_device(ctx, buf, so, sl, want_t, do, caps, want_res)
        out = torch.full((total + 64,), CANARY, dtype=torch.uint8, device="cuda")
        _, res = _outs(n, kind)
        batch.unwrap_to_device_async(ctx, _pinned_bytes(buf), so, sl, out, do, caps, res)
        torch.cuda.synchronize()
    got_res = res.cpu().numpy()
    assert got_res.tolist() == want_res.tolist()
    if which == "statuses":
        assert {E_ARG, E_FORMAT} <= set(want_res.tolist()) and 0 in want_res
    got, want = out.cpu().numpy(), want_t.cpu().numpy()
    slot = np.zeros(len(got), bool)
    for o, c in zip(do, caps):
        slot[o:o + c] = True
    assert (got[~slot] == CANARY).all(), "a device byte outside [dst_off, dst_off + dst_cap) changed"
    for o, r in zip(do, want_res):
        if r >= 0:
            assert got[o:o + r].tobytes() == want[o:o + r].tobytes()


# ---- packed Unwrap, packed decode -----------------------------------------------------------------------------------
def _packed_case(ctx, which):
    """(sources, the synchronous call(ctx, buf, so, sl, out, off, res), the asynchronous one): packets with bad headers
    between good ones, or compressed blocks with a malformed one."""
    from lz4net_b200 import batch
    if which == "unwrap":
        packets, _ = _packets(ctx)
        bad = [b"", b"\x01\x02\x03", struct.pack("<ii", 10, 50) + bytes(5), struct.pack("<Ii", 2 ** 31 + 5, 3) + bytes(3)]
        srcs = [x for i, p in enumerate(packets) for x in ([p, bad[i % 4]] if i % 5 == 2 else [p])]
        return srcs, batch.unwrap_to_device_packed, batch.unwrap_to_device_packed_async
    srcs = [(oracle.encode_hc if i % 2 and len(d) <= 65547 else oracle.encode)(d)[1] for i, d in enumerate(_blocks())]
    srcs.insert(7, b"\xf0\xff\xff\xff")                                  # a literal run past the end: malformed
    return srcs, batch.decode_from_host_packed, batch.decode_from_host_packed_async


def _packed_sync(ctx, call, buf, so, sl, room):
    import torch
    n = len(so)
    out = torch.full((room + 64,), CANARY, dtype=torch.uint8, device="cuda")
    off, res = np.full(n + 1, -7, np.int64), np.full(n, 12345, np.int32)
    call(ctx, buf, so, sl, out[:room], off, res)
    return res, off, out.cpu().numpy()


def _packed_async(ctx, call, buf, so, sl, room, kind):
    import torch
    n = len(so)
    out = torch.full((room + 64,), CANARY, dtype=torch.uint8, device="cuda")
    off, res = _outs(n, kind)
    call(ctx, _pinned_bytes(buf), so, sl, out[:room], off, res)
    torch.cuda.synchronize()
    return res.cpu().numpy(), off.cpu().numpy(), out.cpu().numpy()


@pytest.mark.parametrize("kind", ["device", "pinned"])
@pytest.mark.parametrize("which", ["unwrap", "decode"])
def test_gpu_async_packed_calls_equal_the_synchronous_calls(ctx, which, kind):
    srcs, sync, async_ = _packed_case(ctx, which)
    buf, so, sl = _src(srcs, skew=1, gap=2)
    with _Options(ctx, host_chunk_mb=1):
        want_res, want_off, _ = _packed_sync(ctx, sync, buf, so, sl, 1)             # sizes only: the total
        total = int(want_off[-1])
        want_res, want_off, want = _packed_sync(ctx, sync, buf, so, sl, total)
        res, off, got = _packed_async(ctx, async_, buf, so, sl, total, kind)
    assert res.tolist() == want_res.tolist() and np.array_equal(off, want_off)
    assert (want_res < 0).sum() >= 1 and (want_res >= 0).sum() > 20
    assert (got[total:] == CANARY).all()
    for o, r in zip(off, res):
        if r >= 0:
            assert got[o:o + r].tobytes() == want[o:o + r].tobytes()


@pytest.mark.parametrize("which", ["unwrap", "decode"])
def test_gpu_async_packed_calls_into_a_destination_too_small(ctx, which):
    srcs, sync, async_ = _packed_case(ctx, which)
    buf, so, sl = _src(srcs, skew=1, gap=2)
    with _Options(ctx, host_chunk_mb=1):
        want_res, want_off, _ = _packed_sync(ctx, sync, buf, so, sl, 1)
        total = int(want_off[-1])
        for short in (1, total // 2, total - 1):
            res, off, got = _packed_async(ctx, async_, buf, so, sl, total - short, "pinned")
            assert np.array_equal(off, want_off), short
            # non-negative exactly for the well-formed ones, where it is the size
            assert ((res >= 0) == (want_res >= 0)).all(), short
            assert (res[res >= 0] == want_res[want_res >= 0]).all(), short
            assert (got[total - short:] == CANARY).all(), short               # nothing behind dst_total_cap


def test_gpu_async_unwrap_reads_headers_that_queued_work_writes(ctx):
    """The pinned buffer holds bytes whose headers are all E_FORMAT when the calls are made; an asynchronous Wrap queued
    behind a sleep writes the packets, and the asynchronous packed Unwrap enqueued right after it must restore them."""
    import torch
    from lz4net_b200 import batch
    blocks = _blocks()
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    want_res, want_off, want = _sync_wrap(ctx, raw, so, sl, False)
    wire = _pinned(int(want_off[-1]), 0xFF)                            # rawLen = -1 everywhere
    plain = np.concatenate([np.frombuffer(b, np.uint8) for b in blocks])
    s = torch.cuda.Stream()
    with _Options(ctx, host_chunk_mb=1), torch.cuda.stream(s):
        off, res = _outs(n, "device")
        back = torch.full((len(plain) + 64,), CANARY, dtype=torch.uint8, device="cuda")
        back_off, back_len = _outs(n, "device")
        torch.cuda._sleep(100_000_000)
        batch.wrap_to_host_packed_async(ctx, raw, so, sl, wire, off, res)
        batch.unwrap_to_device_packed_async(ctx, wire, want_off[:n].copy(), want_res, back[:len(plain)], back_off, back_len)
        s.synchronize()
    assert wire.numpy().tobytes() == want
    assert back_len.cpu().tolist() == [len(b) for b in blocks]
    assert back.cpu().numpy()[:len(plain)].tobytes() == plain.tobytes() and (back.cpu().numpy()[len(plain):] == CANARY).all()


def test_gpu_async_packed_calls_of_no_blocks_write_the_total(ctx):
    import torch
    from lz4net_b200 import batch
    raw = torch.zeros(16, dtype=torch.uint8, device="cuda")
    e = np.zeros(0, np.int64)
    for kind in ("device", "pinned"):
        for call in (lambda o, r: batch.wrap_to_host_packed_async(ctx, raw, e, e.astype(np.int32), _pinned(16, 0), o, r),
                     lambda o, r: batch.unwrap_to_device_packed_async(ctx, _pinned(16, 0), e, e.astype(np.int32), raw, o, r),
                     lambda o, r: batch.decode_from_host_packed_async(ctx, _pinned(16, 0), e, e.astype(np.int32), raw, o, r)):
            off, res = _outs(0, kind)
            call(off, res)
            torch.cuda.synchronize()
            assert off.cpu().tolist() == [0]


# ---- non-blocking, ordering --------------------------------------------------------------------------------------------
def test_gpu_async_calls_return_while_the_stream_is_busy(ctx):
    import torch
    from lz4net_b200 import batch
    packets, blocks = _packets(ctx)
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    wbuf, wso, wsl = _src(packets)
    wire = _pinned_bytes(wbuf)
    comp = [oracle.encode(d)[1] for d in blocks]
    cbuf, cso, csl = _src(comp)
    cpin = _pinned_bytes(cbuf)
    do, total = _layout(sl, 3, 5)
    s = torch.cuda.Stream()
    dst = _pinned(int(sl.sum()) + 8 * n, 0)
    out = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    off, res = _outs(n, "device")
    calls = {
        "wrap": lambda: batch.wrap_to_host_packed_async(ctx, raw, so, sl, dst, off, res),
        "unwrap": lambda: batch.unwrap_to_device_async(ctx, wire, wso, wsl, out, do, sl, res),
        "unwrap packed": lambda: batch.unwrap_to_device_packed_async(ctx, wire, wso, wsl, out, off, res),
        "decode packed": lambda: batch.decode_from_host_packed_async(ctx, cpin, cso, csl, out, off, res),
    }
    for warm in (True, False):
        for name, call in calls.items():
            with torch.cuda.stream(s):
                if not warm:
                    torch.cuda._sleep(300_000_000)
                call()
                if not warm:
                    assert not s.query(), f"the {name} waited for the device"
                s.synchronize()
                assert (res.cpu().numpy() >= 0).all(), name
    plain = np.concatenate([np.frombuffer(b, np.uint8) for b in blocks])
    assert out.cpu().numpy()[:len(plain)].tobytes() == plain.tobytes()          # the packed decode, last
    assert off.cpu().tolist() == [0] + np.cumsum(sl).tolist()


def test_gpu_async_wrap_and_unwrap_are_ordered_on_the_callers_stream_and_between_streams(ctx):
    """Per stream: a kernel filling the inputs, the asynchronous Wrap into a pinned buffer, the asynchronous packed Unwrap
    out of it (packet offsets from an earlier synchronous Wrap of the same data) and a consumer of its results, all
    enqueued behind a sleep; two streams with one context."""
    import torch
    from lz4net_b200 import batch, synth
    n, bs = 64, 65536
    want_raw = np.concatenate([synth.make_blocks(c, n // 4, bs, seed=7, first_block=k * (n // 4)).reshape(-1)
                               for k, c in enumerate(synth.CLASSES)])
    so = np.arange(n, dtype=np.int64) * bs
    sl = np.full(n, bs, np.int32)
    want_res, want_off, want = _sync_wrap(ctx, _dev(want_raw), so, sl, False)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    raws = [torch.zeros(n * bs, dtype=torch.uint8, device="cuda") for _ in streams]
    wires = [_pinned(int(want_off[-1]), 0xFF) for _ in streams]
    backs = [torch.zeros(n * bs, dtype=torch.uint8, device="cuda") for _ in streams]
    copies = []
    with _Options(ctx, host_chunk_mb=1):
        for s, raw, wire, back in zip(streams, raws, wires, backs):
            with torch.cuda.stream(s):
                off, res = _outs(n, "device")
                boff, blen = _outs(n, "pinned")
                torch.cuda._sleep(50_000_000)
                for k, c in enumerate(synth.CLASSES):                  # the producer: enqueued, not yet run
                    batch.synth_fill(ctx, raw[k * (n // 4) * bs:], n // 4, bs, synth.CLASS_ID[c], seed=7, first_block=k * (n // 4))
                batch.wrap_to_host_packed_async(ctx, raw, so, sl, wire, off, res)
                batch.unwrap_to_device_packed_async(ctx, wire, want_off[:n].copy(), want_res, back, boff, blen)
                copies.append((off.clone(), res.clone(), back.clone(), boff, blen, off, res))  # the consumer
        torch.cuda.synchronize()
    for wire, (off, res, back, boff, blen, _, _) in zip(wires, copies):
        assert res.cpu().tolist() == want_res.tolist() and off.cpu().tolist() == want_off.tolist()
        assert wire.numpy().tobytes() == want
        assert blen.numpy().tolist() == [bs] * n and boff.numpy().tolist() == (np.arange(n + 1) * bs).tolist()
        assert back.cpu().numpy().tobytes() == want_raw.tobytes()


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_gpu_async_calls_refuse_wrong_memory_and_negative_lengths(ctx):
    import torch
    from lz4net_b200 import native
    lib = native.lib()
    d = cases.content("ETEXT", 4096, seed=1).tobytes()
    so, sl = np.zeros(1, np.int64), np.array([len(d)], np.int32)
    neg = np.array([-1], np.int32)
    raw = _dev(np.frombuffer(d, np.uint8))
    off, res = _outs(1, "pinned")
    pk = _pinned(8192, CANARY)
    out = torch.full((8192,), CANARY, dtype=torch.uint8, device="cuda")
    pageable, device = np.full(8192, CANARY, np.uint8), torch.full((8192,), CANARY, dtype=torch.uint8, device="cuda")
    cap = np.array([8192], np.int32)

    def wrap(dst, lens=sl):
        return lib.lz4b200_wrap_batch_packed_from_device_async(ctx.handle, raw.data_ptr(), so.ctypes.data, lens.ctypes.data, 0, dst,
                                                               8192, off.data_ptr(), res.data_ptr(), 1, 0)

    def unwrap(src, lens=sl, caps=cap):
        return lib.lz4b200_unwrap_batch_to_device_async(ctx.handle, src, so.ctypes.data, lens.ctypes.data, out.data_ptr(),
                                                        so.ctypes.data, caps.ctypes.data, res.data_ptr(), 1, 0)

    def unwrap_packed(src, lens=sl):
        return lib.lz4b200_unwrap_batch_packed_to_device_async(ctx.handle, src, so.ctypes.data, lens.ctypes.data, out.data_ptr(),
                                                               8192, off.data_ptr(), res.data_ptr(), 1, 0)

    def decode_packed(src, lens=sl):
        return lib.lz4b200_decode_batch_packed_to_device_async(ctx.handle, src, so.ctypes.data, lens.ctypes.data, out.data_ptr(),
                                                               8192, off.data_ptr(), res.data_ptr(), 1, 0)

    for ptr, name in ((pageable.ctypes.data, "pageable"), (device.data_ptr(), "device")):
        assert wrap(ptr) == E_ARG and "dst" in native.last_error(), name
        for call in (unwrap, unwrap_packed, decode_packed):
            assert call(ptr) == E_ARG and "src" in native.last_error(), (call.__name__, name)
    for call in (wrap, unwrap, unwrap_packed, decode_packed):
        assert call(pk.data_ptr(), lens=neg) == E_ARG and "negative" in native.last_error(), call.__name__
    assert unwrap(pk.data_ptr(), caps=neg) == E_ARG
    # out_off / out_len in pageable memory
    po = np.full(2, -7, np.int64)
    rc = lib.lz4b200_unwrap_batch_packed_to_device_async(ctx.handle, pk.data_ptr(), so.ctypes.data, sl.ctypes.data, out.data_ptr(),
                                                         8192, po.ctypes.data, res.data_ptr(), 1, 0)
    assert rc == E_ARG and "out_off" in native.last_error()
    torch.cuda.synchronize()
    assert off.numpy().tolist() == [-7, -7] and res.numpy().tolist() == [12345] and po.tolist() == [-7, -7]
    assert (out.cpu().numpy() == CANARY).all() and (pk.numpy() == CANARY).all()


def test_gpu_async_calls_refuse_a_capturing_stream_and_leave_the_capture_valid(ctx):
    import torch
    from lz4net_b200 import native
    lib = native.lib()
    d = cases.content("E50", 8192, seed=2).tobytes()
    so, sl, cap = np.zeros(1, np.int64), np.array([len(d)], np.int32), np.array([len(d)], np.int32)
    csl = np.array([10], np.int32)
    raw = _dev(np.frombuffer(d, np.uint8))
    dst, pk = _pinned(len(d) + 8, 0), _pinned(64, 0)
    off, res = _outs(1, "device")
    out = torch.zeros(len(d), dtype=torch.uint8, device="cuda")
    x = torch.zeros(4, device="cuda")
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    rcs = []
    with torch.cuda.graph(g, stream=s):
        st = torch.cuda.current_stream().cuda_stream
        rcs.append(lib.lz4b200_wrap_batch_packed_from_device_async(ctx.handle, raw.data_ptr(), so.ctypes.data, sl.ctypes.data, 1,
                                                                   dst.data_ptr(), dst.numel(), off.data_ptr(), res.data_ptr(), 1, st))
        rcs.append(lib.lz4b200_unwrap_batch_to_device_async(ctx.handle, pk.data_ptr(), so.ctypes.data, csl.ctypes.data, out.data_ptr(),
                                                            so.ctypes.data, cap.ctypes.data, res.data_ptr(), 1, st))
        rcs.append(lib.lz4b200_unwrap_batch_packed_to_device_async(ctx.handle, pk.data_ptr(), so.ctypes.data, csl.ctypes.data,
                                                                   out.data_ptr(), out.numel(), off.data_ptr(), res.data_ptr(), 1, st))
        rcs.append(lib.lz4b200_decode_batch_packed_to_device_async(ctx.handle, pk.data_ptr(), so.ctypes.data, csl.ctypes.data,
                                                                   out.data_ptr(), out.numel(), off.data_ptr(), res.data_ptr(), 1, st))
        x.add_(1)
    assert rcs == [E_ARG] * 4 and "capturing" in native.last_error()
    g.replay()
    torch.cuda.synchronize()
    assert x.cpu().tolist() == [1.0] * 4
    assert off.cpu().tolist() == [-7, -7] and res.cpu().tolist() == [12345]
