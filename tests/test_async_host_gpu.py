"""The asynchronous offload calls on an H100: lz4b200_encode_batch_packed_from_device_async (device memory encoded back to
back into page-locked host memory, landed by a kernel) and lz4b200_decode_batch_to_device_async (page-locked host memory
decoded into device memory).

Results and bytes must be those of the synchronous calls however many pipeline stages a batch spans; a destination too
small is reported through out_off[n] with nothing written behind its capacity; the calls return while the device is still
busy, are ordered on the caller's stream, refuse the wrong kind of memory and a capturing stream."""
import functools

import numpy as np
import pytest

import oracle
from tests import cases
from tests.test_mixed_memory_gpu import _dev, _layout, _Options, _src

pytestmark = pytest.mark.gpu

CLASSES = ("E0", "E50", "E100", "ETEXT")
SIZES = (0, 1, 13, 65536, 65547, 1 << 20)
CANARY = 0x5C
E_ARG = -1


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@functools.lru_cache(maxsize=None)
def _blocks():
    return tuple(cases.content(m, n, seed=40 + i).tobytes() for i, m in enumerate(CLASSES) for n in SIZES)


def _pinned(n, fill, dtype=None):
    import torch
    return torch.full((n,), fill, dtype=dtype or torch.uint8).pin_memory()


def _outs(n, kind):
    """out_off (int64[n+1]) and out_len (int32[n]) in device memory or page-locked host memory, filled with junk."""
    import torch
    if kind == "device":
        return (torch.full((n + 1,), -7, dtype=torch.int64, device="cuda"), torch.full((n,), 12345, dtype=torch.int32, device="cuda"))
    return _pinned(n + 1, -7, torch.int64), _pinned(n, 12345, torch.int32)


def _caps(blocks):
    """The bound for most blocks; every fifth gets its input length (an incompressible block then does not fit: 0 bytes)."""
    return np.array([len(b) if i % 5 == 4 else oracle.bound(len(b)) for i, b in enumerate(blocks)], np.int32)


def _sync_encode(ctx, raw, so, sl, caps, hc):
    from lz4net_b200 import batch
    n = len(so)
    dst = np.zeros(int(caps.sum()) + 64, np.uint8)
    off, res = np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
    total = batch.encode_to_host_packed(ctx, raw, so, sl, caps, dst, off, res, hc=hc)
    return res, off, dst[:total].tobytes()


# ---- parity with the synchronous calls ----------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["device", "pinned"])
@pytest.mark.parametrize("hc", [False, True], ids=["fast", "hc"])
def test_gpu_async_encode_equals_the_synchronous_packed_encode(ctx, hc, kind):
    import torch
    from lz4net_b200 import batch
    blocks = _blocks()
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    caps = _caps(blocks)
    with _Options(ctx, host_chunk_mb=1):                              # every 1 MiB block a stage of its own: more stages than buffers
        want_res, want_off, want = _sync_encode(ctx, raw, so, sl, caps, hc)
        total = int(want_off[-1])
        dst = _pinned(total + 256, CANARY)
        off, res = _outs(n, kind)
        batch.encode_to_host_packed_async(ctx, raw, so, sl, caps, dst, off, res, hc=hc)
        torch.cuda.synchronize()
    assert res.cpu().numpy().tolist() == want_res.tolist()
    assert np.array_equal(off.cpu().numpy(), want_off)
    h = dst.numpy()
    assert h[:total].tobytes() == want and (h[total:] == CANARY).all()


def _decode_case(known):
    """(compressed, capacity, raw): every block fast- or HC-encoded by the oracle; an unknown-size decode gets room."""
    out = []
    for i, d in enumerate(_blocks()):
        c = (oracle.encode_hc if i % 2 and len(d) <= 65547 else oracle.encode)(d)[1]
        out.append((c, len(d) if known else len(d) + 7 * (i % 3), d))
    return out


@pytest.mark.parametrize("kind", ["device", "pinned"])
@pytest.mark.parametrize("known", [True, False], ids=["known", "unknown"])
def test_gpu_async_decode_equals_the_synchronous_decode(ctx, known, kind):
    import torch
    from lz4net_b200 import batch
    case = _decode_case(known)
    comp = [c for c, _, _ in case]
    caps = np.array([k for _, k, _ in case], np.int32)
    buf, so, sl = _src(comp, skew=5, gap=3)
    do, total = _layout(caps, 11, 13)
    with _Options(ctx, host_chunk_mb=1):
        want_t = torch.full((total + 64,), CANARY, dtype=torch.uint8, device="cuda")
        want_res = np.zeros(len(comp), np.int32)
        batch.decode_from_host(ctx, buf, so, sl, want_t, do, caps, want_res, known=known)
        src = _pinned(len(buf), 0)
        src.numpy()[:] = buf
        out = torch.full((total + 64,), CANARY, dtype=torch.uint8, device="cuda")
        _, res = _outs(len(comp), kind)
        batch.decode_from_host_async(ctx, src, so, sl, out, do, caps, res, known=known)
        torch.cuda.synchronize()
    assert res.cpu().numpy().tolist() == want_res.tolist()
    assert all(r >= 0 for r, (_, _, d) in zip(want_res, case) if d)
    got, want = out.cpu().numpy(), want_t.cpu().numpy()
    assert np.array_equal(got, want)                                   # the slots and the canaries around every one of them
    for (_, _, d), o in zip(case, do):
        assert got[o:o + len(d)].tobytes() == d


def test_gpu_async_round_trip_through_one_pinned_buffer(ctx):
    import torch
    from lz4net_b200 import batch
    blocks = _blocks()
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    caps = np.array([oracle.bound(len(b)) for b in blocks], np.int32)
    dst = _pinned(int(caps.sum()), 0)
    off, res = _outs(n, "pinned")
    with _Options(ctx, host_chunk_mb=2):
        batch.encode_to_host_packed_async(ctx, raw, so, sl, caps, dst, off, res, hc=True)
        torch.cuda.synchronize()
        o, r = off.numpy().copy(), res.numpy().copy()
        back = torch.zeros(len(buf), dtype=torch.uint8, device="cuda")
        out_len = torch.zeros(n, dtype=torch.int32, device="cuda")
        batch.decode_from_host_async(ctx, dst, o[:n].copy(), r, back, so, sl, out_len, known=True)
        torch.cuda.synchronize()
    got = out_len.cpu().numpy()
    assert all(g == c for g, c, b in zip(got, r, blocks) if b)          # a known-size decode reads every compressed byte
    assert back.cpu().numpy().tobytes() == buf.tobytes()


def test_gpu_async_encode_into_a_destination_too_small(ctx):
    import torch
    from lz4net_b200 import batch
    blocks = _blocks()
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    caps = np.array([oracle.bound(len(b)) for b in blocks], np.int32)
    with _Options(ctx, host_chunk_mb=1):
        want_res, want_off, want = _sync_encode(ctx, raw, so, sl, caps, False)
        total = int(want_off[-1])
        for short in (1, total // 2, total - 1):
            alloc = _pinned(total + 4096, CANARY)
            off, res = _outs(n, "pinned")
            batch.encode_to_host_packed_async(ctx, raw, so, sl, caps, alloc[:total - short], off, res)
            torch.cuda.synchronize()
            assert res.numpy().tolist() == want_res.tolist() and np.array_equal(off.numpy(), want_off)
            h = alloc.numpy()
            assert (h[total - short:] == CANARY).all(), short             # nothing behind dst_total_cap


def test_gpu_async_encode_of_no_blocks_writes_the_total(ctx):
    import torch
    from lz4net_b200 import batch
    raw = torch.zeros(16, dtype=torch.uint8, device="cuda")
    e = np.zeros(0, np.int64)
    for kind in ("device", "pinned"):
        off, res = _outs(0, kind)
        batch.encode_to_host_packed_async(ctx, raw, e, e.astype(np.int32), e.astype(np.int32), _pinned(16, 0), off, res)
        torch.cuda.synchronize()
        assert off.cpu().tolist() == [0]


# ---- non-blocking, ordering --------------------------------------------------------------------------------------------
def test_gpu_async_calls_return_while_the_stream_is_busy(ctx):
    import torch
    from lz4net_b200 import batch
    blocks = _blocks()
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    caps = np.array([oracle.bound(len(b)) for b in blocks], np.int32)
    want_res, want_off, want = _sync_encode(ctx, raw, so, sl, caps, False)
    total = int(want_off[-1])
    s = torch.cuda.Stream()
    dst = _pinned(total, 0)
    off, res = _outs(n, "device")
    back = torch.zeros(len(buf), dtype=torch.uint8, device="cuda")
    out_len = torch.zeros(n, dtype=torch.int32, device="cuda")
    for warm in (True, False):
        with torch.cuda.stream(s):
            if not warm:
                torch.cuda._sleep(300_000_000)
            batch.encode_to_host_packed_async(ctx, raw, so, sl, caps, dst, off, res)
            if not warm:
                assert not s.query(), "the encode waited for the device"
            s.synchronize()
            assert np.array_equal(off.cpu().numpy(), want_off) and dst.numpy().tobytes() == want
            if not warm:
                torch.cuda._sleep(300_000_000)
            batch.decode_from_host_async(ctx, dst, want_off[:n].copy(), want_res, back, so, sl, out_len, known=True)
            if not warm:
                assert not s.query(), "the decode waited for the device"
            s.synchronize()
            assert back.cpu().numpy().tobytes() == buf.tobytes()
            back.zero_()
            off.fill_(-7)
            dst.zero_()


def test_gpu_async_calls_are_ordered_on_the_callers_stream_and_between_streams(ctx):
    """A kernel filling the source before the call and a consumer after it on the same stream see the right data; two
    calls of one context on two streams both land correctly."""
    import torch
    from lz4net_b200 import batch, synth
    n, bs = 64, 65536
    want_raw = np.concatenate([synth.make_blocks(c, n // 4, bs, seed=5, first_block=k * (n // 4)).reshape(-1)
                               for k, c in enumerate(synth.CLASSES)])
    so = np.arange(n, dtype=np.int64) * bs
    sl = np.full(n, bs, np.int32)
    caps = np.full(n, oracle.bound(bs), np.int32)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    raws = [torch.zeros(n * bs, dtype=torch.uint8, device="cuda") for _ in streams]
    dsts = [_pinned(int(caps.sum()), 0) for _ in streams]
    outs = [_outs(n, "device") for _ in streams]
    copies = []
    with _Options(ctx, host_chunk_mb=1):
        for s, raw, dst, (off, res) in zip(streams, raws, dsts, outs):
            with torch.cuda.stream(s):
                torch.cuda._sleep(50_000_000)
                for k, c in enumerate(synth.CLASSES):                  # the producer: enqueued, not yet run
                    batch.synth_fill(ctx, raw[k * (n // 4) * bs:], n // 4, bs, synth.CLASS_ID[c], seed=5, first_block=k * (n // 4))
                batch.encode_to_host_packed_async(ctx, raw, so, sl, caps, dst, off, res)
                copies.append((off.clone(), res.clone()))            # the consumer: after the call on the same stream
        torch.cuda.synchronize()
    assert raws[0].cpu().numpy().tobytes() == want_raw.tobytes()
    want = ctx.encode_blocks_packed([want_raw[i * bs:(i + 1) * bs].tobytes() for i in range(n)], caps=caps)
    for dst, (off, res) in zip(dsts, copies):
        assert res.cpu().tolist() == list(want[0]) and off.cpu().tolist() == list(want[1])
        assert dst.numpy()[:want[1][-1]].tobytes() == bytes(want[2])


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_gpu_async_calls_refuse_the_wrong_kind_of_memory(ctx):
    import torch
    from lz4net_b200 import native
    lib = native.lib()
    d = cases.content("ETEXT", 4096, seed=1).tobytes()
    comp = oracle.encode(d)[1]
    so, sl, caps = np.zeros(1, np.int64), np.array([len(d)], np.int32), np.array([oracle.bound(len(d))], np.int32)
    raw = _dev(np.frombuffer(d, np.uint8))
    off, res = _outs(1, "pinned")
    for dst, name in ((np.full(8192, CANARY, np.uint8), "pageable"), (torch.full((8192,), CANARY, dtype=torch.uint8, device="cuda"), "device")):
        ptr = dst.ctypes.data if isinstance(dst, np.ndarray) else dst.data_ptr()
        rc = lib.lz4b200_encode_batch_packed_from_device_async(ctx.handle, raw.data_ptr(), so.ctypes.data, sl.ctypes.data,
                                                               caps.ctypes.data, ptr, 8192, off.data_ptr(), res.data_ptr(), 1,
                                                               native.MODE_FAST, 0)
        assert rc == E_ARG and "dst" in native.last_error(), name
    torch.cuda.synchronize()
    assert off.numpy().tolist() == [-7, -7] and res.numpy().tolist() == [12345]
    out = torch.full((len(d),), CANARY, dtype=torch.uint8, device="cuda")
    csl = np.array([len(comp)], np.int32)
    for src, name in ((np.frombuffer(comp, np.uint8).copy(), "pageable"), (_dev(np.frombuffer(comp, np.uint8)), "device")):
        ptr = src.ctypes.data if isinstance(src, np.ndarray) else src.data_ptr()
        rc = lib.lz4b200_decode_batch_to_device_async(ctx.handle, ptr, so.ctypes.data, csl.ctypes.data, out.data_ptr(), so.ctypes.data,
                                                      sl.ctypes.data, res.data_ptr(), 1, 1, 0)
        assert rc == E_ARG and "src" in native.last_error(), name
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == CANARY).all() and res.numpy().tolist() == [12345]


def test_gpu_async_calls_refuse_a_capturing_stream_and_leave_the_capture_valid(ctx):
    import torch
    from lz4net_b200 import native
    lib = native.lib()
    d = cases.content("E50", 8192, seed=2).tobytes()
    so, sl, caps = np.zeros(1, np.int64), np.array([len(d)], np.int32), np.array([oracle.bound(len(d))], np.int32)
    csl = np.array([10], np.int32)
    raw = _dev(np.frombuffer(d, np.uint8))
    dst, comp = _pinned(int(caps[0]), 0), _pinned(64, 0)
    off, res = _outs(1, "device")
    out = torch.zeros(len(d), dtype=torch.uint8, device="cuda")
    x = torch.zeros(4, device="cuda")
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    rcs = []
    with torch.cuda.graph(g, stream=s):
        st = torch.cuda.current_stream().cuda_stream
        rcs.append(lib.lz4b200_encode_batch_packed_from_device_async(ctx.handle, raw.data_ptr(), so.ctypes.data, sl.ctypes.data,
                                                                     caps.ctypes.data, dst.data_ptr(), dst.numel(), off.data_ptr(),
                                                                     res.data_ptr(), 1, native.MODE_FAST, st))
        rcs.append(lib.lz4b200_decode_batch_to_device_async(ctx.handle, comp.data_ptr(), so.ctypes.data, csl.ctypes.data,
                                                            out.data_ptr(), so.ctypes.data, sl.ctypes.data, res.data_ptr(), 1, 1, st))
        x.add_(1)
    assert rcs == [E_ARG, E_ARG] and "capturing" in native.last_error()
    g.replay()
    torch.cuda.synchronize()
    assert x.cpu().tolist() == [1.0] * 4
    assert off.cpu().tolist() == [-7, -7] and res.cpu().tolist() == [12345]
