"""The asynchronous decode and Unwrap from device-written offsets on an H100: lz4b200_decode_batch_to_device_at_async and
lz4b200_unwrap_batch_to_device_at_async restore an offload straight from the out_off that the asynchronous packed encode
or Wrap wrote on the device, with no synchronisation in between.

The round trip must give back the source bytes, and the same out_len and bytes as the host-offset calls given the
offsets read after a synchronise, however many stages the batch spans and wherever src_off lives.  The calls must not
block the caller, must be ordered behind the offload on another stream by the context's chain, must reject each kind of
malformed span (and every block of an offload that did not fit) with LZ4B200_E_ARG and nothing written, and must refuse
a capturing stream.  Every out-of-range offset used here lies inside the page-locked allocation, so a faulty bound check
shows up as a wrong status or wrong bytes."""
import numpy as np
import pytest

from tests import cases
from tests.test_mixed_memory_gpu import _dev, _layout, _Options, _src

pytestmark = pytest.mark.gpu

CLASSES = ("E0", "E50", "E100", "ETEXT")
SIZES = (0, 1, 65536, 200 * 1024)                                        # 200 KiB: the HC encoder's large-block path
CANARY = 0x5C
E_ARG = -1
SKEW = 3                                                                 # the page-locked base is not 16-byte aligned


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


def _blocks():
    return [cases.content(m, n, seed=90 + i).tobytes() for i, m in enumerate(CLASSES) for n in SIZES]


def _bound(n):
    return n + n // 255 + 16


def _pinned(n, fill, dtype=None):
    import torch
    return torch.full((n,), fill, dtype=dtype or torch.uint8).pin_memory()


def _offsets(n, where):
    """out_off (int64[n+1]) in device memory or page-locked host memory, and out_len (int32[n]) on the device."""
    import torch
    off = torch.full((n + 1,), -7, dtype=torch.int64, device="cuda") if where == "device" else _pinned(n + 1, -7, torch.int64)
    return off, torch.full((n,), 12345, dtype=torch.int32, device="cuda")


def _offload(ctx, wrap, raw, so, sl, hc, dst, off, res, stream=None):
    from lz4net_b200 import batch
    if wrap:
        batch.wrap_to_host_packed_async(ctx, raw, so, sl, dst, off, res, hc=hc, stream=stream)
    else:
        caps = np.array([_bound(int(x)) for x in sl], np.int32)
        batch.encode_to_host_packed_async(ctx, raw, so, sl, caps, dst, off, res, hc=hc, stream=stream)


def _restore(ctx, wrap, src, src_cap, src_off, out, dst_off, dst_cap, out_len, known=True, stream=None):
    from lz4net_b200 import batch
    if wrap:
        batch.unwrap_to_device_at_async(ctx, src, src_cap, src_off, out, dst_off, dst_cap, out_len, stream=stream)
    else:
        batch.decode_from_host_at_async(ctx, src, src_cap, src_off, out, dst_off, dst_cap, out_len, known=known, stream=stream)


def _host_form(ctx, wrap, src, off, out, dst_off, dst_cap, known):
    """The host-offset call over the offsets read on the host: (out_len, out bytes)."""
    import torch
    from lz4net_b200 import batch
    so, sl = off[:-1].copy(), np.diff(off).astype(np.int32)
    res = torch.full((len(sl),), 12345, dtype=torch.int32, device="cuda")
    if wrap:
        batch.unwrap_to_device_async(ctx, src, so, sl, out, dst_off, dst_cap, res)
    else:
        batch.decode_from_host_async(ctx, src, so, sl, out, dst_off, dst_cap, res, known=known)
    torch.cuda.synchronize()
    return res.cpu().numpy(), out.cpu().numpy()


def _round_trip(ctx, wrap, hc, known, where):
    import torch
    blocks = _blocks()
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    cap = int(sl.sum()) + 8 * n if wrap else sum(_bound(int(x)) for x in sl)
    alloc = _pinned(SKEW + cap + 64, CANARY)
    dst = alloc[SKEW:SKEW + cap]
    off, res = _offsets(n, where)
    back = torch.full((buf.size + 64,), CANARY, dtype=torch.uint8, device="cuda")
    back_len = torch.full((n,), 12345, dtype=torch.int32, device="cuda")
    with _Options(ctx, host_chunk_mb=1):                                  # several stages on both sides
        _offload(ctx, wrap, raw, so, sl, hc, dst, off, res)
        _restore(ctx, wrap, dst, cap, off, back, so, sl, back_len, known=known)          # no synchronisation in between
        torch.cuda.synchronize()
        got = back.cpu().numpy()
        for i, b in enumerate(blocks):
            assert got[so[i]:so[i] + len(b)].tobytes() == b, i
        host_off = off.cpu().numpy()
        assert host_off[-1] <= cap
        want_len, want = _host_form(ctx, wrap, dst, host_off, torch.full_like(back, CANARY), so, sl, known)
    assert back_len.cpu().numpy().tolist() == want_len.tolist()
    assert np.array_equal(got, want)


@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("known", [1, 0], ids=["known", "unknown"])
@pytest.mark.parametrize("hc", [False, True], ids=["fast", "hc"])
def test_gpu_codec_round_trip_with_no_host_wait(ctx, hc, known, where):
    _round_trip(ctx, False, hc, known, where)


@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("hc", [False, True], ids=["fast", "hc"])
def test_gpu_wrap_round_trip_with_no_host_wait(ctx, hc, where):
    _round_trip(ctx, True, hc, 1, where)


# ---- non-blocking, ordering --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wrap", [False, True], ids=["codec", "wrap"])
def test_gpu_the_round_trip_does_not_block_the_caller(ctx, wrap):
    """The offload and the restore behind a sleep on one stream; then the offload on one stream and the restore on another,
    which only the context's chain orders behind it."""
    import torch
    n, bs = 64, 65536
    blocks = [cases.content(CLASSES[i % 4], bs, seed=300 + i).tobytes() for i in range(n)]
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    cap = int(sl.sum()) + 8 * n if wrap else sum(_bound(int(x)) for x in sl)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for warm, two in ((True, False), (False, False), (False, True)):
        dst = _pinned(cap, 0)
        off, res = _offsets(n, "device")
        back = torch.zeros(buf.size, dtype=torch.uint8, device="cuda")
        back_len = torch.zeros(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(s1):
            if not warm:
                torch.cuda._sleep(300_000_000)
            _offload(ctx, wrap, raw, so, sl, False, dst, off, res, stream=s1)
        _restore(ctx, wrap, dst, cap, off, back, so, sl, back_len, stream=s2 if two else s1)
        if not warm:
            assert not s1.query() and not (s2 if two else s1).query(), "a call waited for the device"
        torch.cuda.synchronize()
        # a known-size decode reports the bytes it read, an Unwrap the bytes it restored
        assert back_len.cpu().tolist() == (sl.tolist() if wrap else np.diff(off.cpu().numpy()).tolist()), (warm, two)
        got = back.cpu().numpy()
        assert all(got[so[i]:so[i] + len(b)].tobytes() == b for i, b in enumerate(blocks)), (warm, two)


# ---- rejected spans ----------------------------------------------------------------------------------------------------
def _hand_made(ctx, wrap):
    """Four real blocks (compressed, or packets) placed by hand, and a src_off of nine blocks in which five spans are
    malformed: (alloc, src_cap, src_off, dst_cap, the index of each real block, the raw blocks, their out_len)."""
    import torch
    from lz4net_b200 import batch
    raws = [cases.content(c, 5000 + 1000 * i, seed=40 + i).tobytes() for i, c in enumerate(("E50", "ETEXT", "E100", "E0"))]
    buf, so, sl = _src(raws)
    dst = np.zeros(int(sl.sum()) + 8 * 4 + 4096, np.uint8)
    off, res = np.zeros(5, np.int64), np.zeros(4, np.int32)
    if wrap:
        batch.wrap_to_host_packed(ctx, _dev(buf), so, sl, dst, off, res)
    else:
        batch.encode_to_host_packed(ctx, _dev(buf), so, sl, np.array([_bound(int(x)) for x in sl], np.int32), dst, off, res)
    torch.cuda.synchronize()
    comp = [dst[off[i]:off[i + 1]].tobytes() for i in range(4)]
    L = [len(c) for c in comp]
    g1 = L[0] + 64
    g2 = g1 + L[1] + 64
    over = 100                                                            # block 7's dst_cap
    bound7 = over + 8 if wrap else _bound(over)
    o8 = g2 + L[2] + bound7 + 1
    src_cap = o8 + L[3] + 32
    # blk0 good | blk1 decreasing | blk2 negative start | blk3 good | blk4 past src_cap | blk5 starting past src_cap,
    # decreasing | blk6 good | blk7 one byte over its bound | blk8 good
    src_off = np.array([0, L[0], -5, g1, g1 + L[1], src_cap + 10, g2, g2 + L[2], o8, o8 + L[3]], np.int64)
    alloc = _pinned(SKEW + src_cap + 8192, 0)
    h = alloc.numpy()[SKEW:]
    h[src_cap:] = np.frombuffer((comp[0] * (8192 // len(comp[0]) + 1))[:h.size - src_cap], np.uint8)   # a valid-looking tail
    for at, c in ((0, comp[0]), (g1, comp[1]), (g2, comp[2]), (o8, comp[3])):
        h[at:at + len(c)] = np.frombuffer(c, np.uint8)
    h[g2 + L[2]:o8] = np.frombuffer((comp[2] * 4)[:o8 - g2 - L[2]], np.uint8)
    dst_cap = np.array([len(raws[0]), 256, 256, len(raws[1]), 1 << 20, 256, len(raws[2]), over, len(raws[3])], np.int32)
    lens = [len(r) for r in raws] if wrap else L                          # a known-size decode reports the bytes it read
    return alloc[SKEW:SKEW + src_cap + 8192], src_cap, src_off, dst_cap, {0: 0, 3: 1, 6: 2, 8: 3}, raws, lens


@pytest.mark.parametrize("where", ["device", "pinned"])
@pytest.mark.parametrize("wrap", [False, True], ids=["codec", "wrap"])
def test_gpu_rejected_spans_report_e_arg_and_write_nothing(ctx, wrap, where):
    import torch
    src, src_cap, src_off, dst_cap, good, raws, lens = _hand_made(ctx, wrap)
    n = len(dst_cap)
    dst_off, total = _layout(dst_cap, 7, 33)
    back = torch.full((total + 64,), CANARY, dtype=torch.uint8, device="cuda")
    res = torch.full((n,), 12345, dtype=torch.int32, device="cuda")
    off = _dev(src_off) if where == "device" else torch.from_numpy(src_off).pin_memory()
    with _Options(ctx, host_chunk_mb=1):
        _restore(ctx, wrap, src, src_cap, off, back, dst_off, dst_cap, res)
        torch.cuda.synchronize()
    got, out = res.cpu().tolist(), back.cpu().numpy()
    for i in range(n):
        d = out[dst_off[i]:dst_off[i] + dst_cap[i]]
        if i in good:
            assert got[i] == lens[good[i]] and d.tobytes() == raws[good[i]], i
        else:
            assert got[i] == E_ARG and (d == CANARY).all(), (i, got[i])
    gaps = np.ones(out.size, bool)
    for o, c in zip(dst_off, dst_cap):
        gaps[o:o + c] = False
    assert (out[gaps] == CANARY).all(), "written outside every block's range"


@pytest.mark.parametrize("wrap", [False, True], ids=["codec", "wrap"])
def test_gpu_an_offload_that_did_not_fit_restores_nothing(ctx, wrap):
    """The offload's destination is a prefix of a larger page-locked allocation that holds valid-looking data behind it;
    out_off[n] exceeds src_cap, so every block is LZ4B200_E_ARG and the device destination keeps its canary."""
    import torch
    blocks = _blocks()
    n = len(blocks)
    buf, so, sl = _src(blocks)
    raw = _dev(buf)
    full = int(sl.sum()) + 8 * n if wrap else sum(_bound(int(x)) for x in sl)
    first = cases.content("E50", 4096, seed=3).tobytes()
    alloc = _pinned(full + 64, 0)
    alloc.numpy()[:] = np.frombuffer((first * (full // len(first) + 2))[:full + 64], np.uint8)
    with _Options(ctx, host_chunk_mb=1):
        for src_cap in (4096, 200_000):                                    # the E0 blocks alone take more
            dst = alloc[:src_cap]
            off, res = _offsets(n, "device")
            back = torch.full((buf.size + 64,), CANARY, dtype=torch.uint8, device="cuda")
            back_len = torch.full((n,), 12345, dtype=torch.int32, device="cuda")
            _offload(ctx, wrap, raw, so, sl, False, dst, off, res)
            _restore(ctx, wrap, dst, src_cap, off, back, so, sl, back_len)
            torch.cuda.synchronize()
            assert int(off[-1]) > src_cap, src_cap
            assert back_len.cpu().tolist() == [E_ARG] * n, src_cap
            assert (back.cpu().numpy() == CANARY).all(), src_cap


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_gpu_calls_refuse_wrong_memory(ctx):
    import torch
    from lz4net_b200 import native
    lib = native.lib()
    pk = _pinned(8192, CANARY)
    out = torch.full((8192,), CANARY, dtype=torch.uint8, device="cuda")
    res = _pinned(1, 12345, torch.int32)
    dof, cap = np.zeros(1, np.int64), np.array([4096], np.int32)
    dev_off, pageable_off = _dev(np.array([0, 10], np.int64)), np.array([0, 10], np.int64)

    def calls(src, src_off, caps=cap):
        yield lib.lz4b200_decode_batch_to_device_at_async(ctx.handle, src, 8192, src_off, out.data_ptr(), dof.ctypes.data,
                                                          caps.ctypes.data, res.data_ptr(), 1, 1, 0)
        yield lib.lz4b200_unwrap_batch_to_device_at_async(ctx.handle, src, 8192, src_off, out.data_ptr(), dof.ctypes.data,
                                                          caps.ctypes.data, res.data_ptr(), 1, 0)

    for rc in calls(np.zeros(64, np.uint8).ctypes.data, dev_off.data_ptr()):
        assert rc == E_ARG and "src" in native.last_error()
    for rc in calls(out.data_ptr(), dev_off.data_ptr()):
        assert rc == E_ARG and "src" in native.last_error()
    for rc in calls(pk.data_ptr(), pageable_off.ctypes.data):
        assert rc == E_ARG and "src_off" in native.last_error()
    for rc in calls(pk.data_ptr(), dev_off.data_ptr(), np.array([-1], np.int32)):
        assert rc == E_ARG and "negative" in native.last_error()
    torch.cuda.synchronize()
    assert res.numpy().tolist() == [12345] and (out.cpu().numpy() == CANARY).all()


def test_gpu_calls_refuse_a_capturing_stream_and_leave_the_capture_valid(ctx):
    import torch
    from lz4net_b200 import native
    lib = native.lib()
    pk = _pinned(64, 0)
    src_off = _dev(np.array([0, 10], np.int64))
    dof, cap = np.zeros(1, np.int64), np.array([64], np.int32)
    res = torch.full((1,), 12345, dtype=torch.int32, device="cuda")
    out = torch.zeros(64, dtype=torch.uint8, device="cuda")
    x = torch.zeros(4, device="cuda")
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    rcs = []
    with torch.cuda.graph(g, stream=s):
        st = torch.cuda.current_stream().cuda_stream
        rcs.append(lib.lz4b200_decode_batch_to_device_at_async(ctx.handle, pk.data_ptr(), 64, src_off.data_ptr(), out.data_ptr(),
                                                               dof.ctypes.data, cap.ctypes.data, res.data_ptr(), 1, 1, st))
        rcs.append(lib.lz4b200_unwrap_batch_to_device_at_async(ctx.handle, pk.data_ptr(), 64, src_off.data_ptr(), out.data_ptr(),
                                                               dof.ctypes.data, cap.ctypes.data, res.data_ptr(), 1, st))
        x.add_(1)
    assert rcs == [E_ARG] * 2 and "capturing" in native.last_error()
    g.replay()
    torch.cuda.synchronize()
    assert x.cpu().tolist() == [1.0] * 4
    assert res.cpu().tolist() == [12345]
