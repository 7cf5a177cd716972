"""The LZ4Stream decode from a size the device wrote (lz4b200_stream_decode_to_device_at_async) on an H100.

The asynchronous stream encode writes the stream's size only on the device; this call reads it there, walks the headers
on the device and decodes, so an offload and its restore are enqueued back to back with no host wait.  The bytes must be
the source's and out_size its length for every class, mode and chunk size, over many stages, with the size in device or
page-locked memory; streams of any writer decode as the synchronous call decodes them; every status matches the
synchronous call's within the three bounds, and each bound gives E_ARG; a size outside [0, src_cap] writes nothing; the
call returns while the device is busy and refuses the wrong memory and a capturing stream."""
import numpy as np
import pytest

from tests.test_async_stream_gpu import (CANARY, CLASSES, E_ARG, E_FORMAT, G, _bound, _chunk, _crafted_equal_length_block, _data,
                                         _good, _pinned, _pinned_bytes, _size_cell, _sync_decode, _sync_encode)
from tests.test_mixed_memory_gpu import _dev, _Options
from tests.test_stream_walk_emu import MALFORMED, expected

pytestmark = pytest.mark.gpu

N = 3 * (1 << 20) + 12345


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


def _restore(ctx, src, src_cap, size, bs, cap, kind="device", stream=None):
    """The call into a device buffer of cap bytes with G canary bytes on both sides.  size: a tensor holding S (its
    first cell), or an int to put in a fresh cell of `kind`.  Returns (rc, out_size cell pair, bytes of cap, canaries)."""
    import torch
    from lz4net_b200 import native
    if isinstance(size, int):
        cell = _size_cell(kind)
        cell[0] = size
        size = cell
    out = torch.full((cap + 2 * G,), CANARY, dtype=torch.uint8, device="cuda")
    res = _size_cell(kind)
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = native.lib().lz4b200_stream_decode_to_device_at_async(ctx.handle, src.data_ptr(), src_cap, size.data_ptr(), bs,
                                                               out.data_ptr() + G, cap, res.data_ptr(), st)
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    return rc, res.cpu().tolist(), o[G:G + cap].tobytes(), np.concatenate([o[:G], o[G + cap:]])


def _round_trip(ctx, data, bs, hc, kind):
    """encode -> this call on one stream, no synchronise in between; returns (out_size, restored bytes, canaries ok)."""
    import torch
    from lz4net_b200 import batch
    n = len(data)
    raw = _dev(np.frombuffer(data, np.uint8)) if n else torch.zeros(0, dtype=torch.uint8, device="cuda")
    cap = _bound(n, bs)
    buf = _pinned(max(cap, 1), 0)
    d_size, d_out = _size_cell(kind), _size_cell(kind)
    y = torch.full((n + 2 * G,), CANARY, dtype=torch.uint8, device="cuda")
    batch.stream_encode_to_host_async(ctx, raw, buf[:cap], d_size, block_size=bs, hc=hc)
    batch.stream_decode_to_device_at_async(ctx, buf, cap, d_size, y[G:G + n], d_out, block_size=bs)
    torch.cuda.synchronize()
    o = y.cpu().numpy()
    return d_out.cpu().tolist(), o[G:G + n].tobytes(), (o[:G] == CANARY).all() and (o[G + n:] == CANARY).all()


@pytest.mark.parametrize("bs", (16, 1000, 65536, 1 << 20, N + 1), ids=lambda b: f"bs{b}")
@pytest.mark.parametrize("hc", [False, True], ids=["fast", "hc"])
@pytest.mark.parametrize("cls", CLASSES)
def test_gpu_round_trip_with_no_host_wait(ctx, cls, hc, bs):
    data = _data(cls) if bs > 16 else _data(cls, 200_000)
    with _Options(ctx, host_chunk_mb=1):                                # many stages
        for kind in ("device", "pinned"):
            size, got, canaries = _round_trip(ctx, data, bs, hc, kind)
            assert size == [len(data), -7], kind
            assert got == data and canaries, kind
    if bs == 65536:
        size, got, canaries = _round_trip(ctx, data, bs, hc, "device")      # the default stage plan
        assert size == [len(data), -7] and got == data and canaries


def test_gpu_round_trip_of_nothing_and_of_tiny_inputs(ctx):
    for n in (0, 1, 15, 16, 17, 100):
        for hc in (False, True):
            size, got, canaries = _round_trip(ctx, _data("ETEXT", 128)[:n], 16, hc, "pinned")
            assert size == [n, -7] and got == _data("ETEXT", 128)[:n] and canaries, (n, hc)


def test_gpu_streams_of_any_writer(ctx):
    """The synchronous encode's stream, and the Python LZ4Stream's with several Write / Flush calls (short chunks)."""
    import io
    import lz4net_b200
    from lz4net_b200 import codec
    data = _data("MIX", 1 << 20)
    raw = _dev(np.frombuffer(data, np.uint8))
    wires = {"sync": _sync_encode(ctx, raw, 65536, False), "sync-hc": _sync_encode(ctx, raw, 4096, True)}
    sink = io.BytesIO()
    with codec.LZ4Stream(sink, codec.LZ4StreamMode.Compress, codec.LZ4StreamFlags.IsolateInnerStream, 65536, batchBlocks=7,
                         context=lz4net_b200.default_context()) as s:
        for a, b in ((0, 100), (100, 70_000), (70_000, 70_001), (70_001, 400_000), (400_000, len(data))):
            s.Write(data, a, b - a)
            s.Flush()
    wires["LZ4Stream"] = sink.getvalue()
    for name, wire in wires.items():
        bs = 4096 if name == "sync-hc" else 65536
        # the flushes add short chunks: K = ceil(dst_cap / block_size) must cover them
        extra = 8 * bs if name == "LZ4Stream" else 0
        if extra:
            rc, size, _, canaries = _restore(ctx, _pinned_bytes(wire), len(wire), len(wire), bs, len(data))
            assert rc == 0 and size == [E_ARG, -7] and (canaries == CANARY).all()
        with _Options(ctx, host_chunk_mb=1):
            for cap in (len(data) + extra, len(data) + extra + 12345):
                rc, size, got, canaries = _restore(ctx, _pinned_bytes(wire), len(wire), len(wire), bs, cap)
                assert rc == 0 and size == [len(data), -7] and got[:len(data)] == data, (name, cap)
                assert (canaries == CANARY).all() and set(got[len(data):]) <= {CANARY}, name


def test_gpu_status_parity_with_the_synchronous_call(ctx):
    """The emulator's malformed corpus and streams whose payloads do not decode: out_size equals what
    lz4b200_stream_decode_to_device returns, within the bounds; nothing is written outside dst."""
    wire, data = _good(ctx)
    eq_data, eq_block = _crafted_equal_length_block()
    streams = dict(MALFORMED)
    streams.update({
        "good": wire,
        "garbage-payload": _chunk(1, 100, b"\xf0"),
        "good-then-garbage": wire + _chunk(1, 100, b"\xf0") + wire,
        "equal-length-compressed": _chunk(1, len(eq_data), eq_block),
        "equal-length-garbage": _chunk(1, 33, bytes(range(33))),
        "stored-then-equal": _chunk(0, 5, b"hello") + _chunk(1, len(eq_data), eq_block),
        "empty-chunks": _chunk(0, 0, b"") * 5 + _chunk(2, 0, b""),
    })
    rng = np.random.default_rng(5)
    for k in range(6):
        w = bytearray(wire)
        for p in rng.integers(len(w) // 4, len(w), 3):
            w[p] ^= 0xFF
        streams[f"corrupt-{k}"] = bytes(w)
    seen = set()
    for name, w in streams.items():
        cap = 2 * len(data) + 400
        want, want_bytes = _sync_decode(ctx, w, cap)
        with _Options(ctx, host_chunk_mb=1):
            rc, size, got, canaries = _restore(ctx, _pinned_bytes(w), len(w), len(w), 65536, cap, "pinned")
        # the walk's own verdict comes first where a chunk breaks a bound before the first malformed header
        walked = expected(w, len(w), len(w), 65536, cap)[0]
        assert rc == 0 and size == [walked if walked < 0 else want, -7], (name, want, walked, size)
        assert (canaries == CANARY).all(), name
        if want >= 0:
            assert got[:want] == want_bytes, name
        seen.add(want if want < 0 else 0)
    assert seen == {0, E_FORMAT}


def test_gpu_each_bound_gives_e_arg(ctx):
    from tests.test_stream_walk_emu import chunk
    s = chunk(8) + chunk(8) + chunk(8)
    src = _pinned_bytes(s)
    for bs, cap, want in ((8, 24, 24), (7, 24, E_ARG), (8, 23, E_ARG), (8, 16, E_ARG), (12, 24, E_ARG)):
        rc, size, got, canaries = _restore(ctx, src, len(s), len(s), bs, cap)
        assert rc == 0 and size == [want, -7] and (canaries == CANARY).all(), (bs, cap)


def test_gpu_source_size_out_of_range_writes_nothing(ctx):
    wire, data = _good(ctx)
    src = _pinned_bytes(wire)
    for S, src_cap in ((len(wire) + 1, len(wire)), (-1, len(wire)), (len(wire), len(wire) - 1), (1, 0)):
        for kind in ("device", "pinned"):
            rc, size, got, canaries = _restore(ctx, src, src_cap, S, 65536, len(data), kind)
            assert rc == 0 and size == [E_ARG, -7] and set(got) == {CANARY} and (canaries == CANARY).all(), (S, src_cap)


def test_gpu_the_call_returns_while_the_stream_is_busy(ctx):
    import torch
    from lz4net_b200 import batch
    data = _data("MIX", 4 << 20)
    raw = _dev(np.frombuffer(data, np.uint8))
    cap = _bound(len(data), 65536)
    buf = _pinned(cap, 0)
    d_size, d_out = _size_cell("device"), _size_cell("device")
    y = torch.zeros(len(data), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    for warm in (True, False):
        with torch.cuda.stream(s):
            if not warm:
                torch.cuda._sleep(300_000_000)
            batch.stream_encode_to_host_async(ctx, raw, buf, d_size, block_size=65536, stream=s)
            batch.stream_decode_to_device_at_async(ctx, buf, cap, d_size, y, d_out, block_size=65536, stream=s)
            if not warm:
                assert not s.query(), "the call waited for the device"
            s.synchronize()
        assert int(d_out[0]) == len(data) and y.cpu().numpy().tobytes() == data


def test_gpu_refusals(ctx):
    import torch
    from lz4net_b200 import batch, native
    lib = native.lib()
    wire, data = _good(ctx)
    src, cell = _pinned_bytes(wire), _size_cell("device")
    cell[0] = len(wire)
    out, res = torch.zeros(len(data), dtype=torch.uint8, device="cuda"), _size_cell("device")
    st = torch.cuda.current_stream().cuda_stream

    def call(s=src.data_ptr(), cap=len(wire), size=cell.data_ptr(), bs=65536, dst=out.data_ptr(), dcap=len(data), r=res.data_ptr()):
        return lib.lz4b200_stream_decode_to_device_at_async(ctx.handle, s, cap, size, bs, dst, dcap, r, st)

    pageable = np.frombuffer(wire, np.uint8).copy()
    dev_src = _dev(np.frombuffer(wire, np.uint8))
    host_out = np.zeros(len(data), np.uint8)
    pageable_cell = np.array([len(wire)], np.int64)
    for args, text in (({"s": pageable.ctypes.data}, "src must be page-locked"), ({"s": dev_src.data_ptr()}, "src must be page-locked"),
                       ({"size": pageable_cell.ctypes.data}, "src_size must be"), ({"dst": host_out.ctypes.data}, "dst must be device"),
                       ({"r": pageable_cell.ctypes.data}, "out_size must be"), ({"cap": -1}, "bad argument"),
                       ({"dcap": -1}, "bad argument"), ({"bs": 0}, "block_size"), ({"bs": (1 << 31) - 11}, "block_size"),
                       ({"s": None}, "null"), ({"size": None}, "null"), ({"r": None}, "null"), ({"dst": None}, "null")):
        assert call(**args) == E_ARG and text in native.last_error(), (args, native.last_error())
    torch.cuda.synchronize()
    assert res.cpu().tolist() == [-7, -7] and int(out.sum()) == 0
    assert call(bs=(1 << 31) - 12) == 0                                    # the largest block_size is accepted ...
    torch.cuda.synchronize()
    assert res.cpu().tolist() == [E_ARG, -7]                               # ... though K = 1 slot is too few for this stream
    assert call(dcap=len(data) + 8 * 65536) == 0
    torch.cuda.synchronize()
    assert res.cpu().tolist() == [len(data), -7]
    with pytest.raises(TypeError, match="wire: expected a page-locked"):
        batch.stream_decode_to_device_at_async(ctx, torch.zeros(8, dtype=torch.uint8), 8, cell, out, res)
    with pytest.raises(TypeError, match="src_size: expected a page-locked"):
        batch.stream_decode_to_device_at_async(ctx, src, len(wire), torch.zeros(1, dtype=torch.int64), out, res)
    with pytest.raises(ValueError, match="src_cap"):
        batch.stream_decode_to_device_at_async(ctx, src, src.numel() + 1, cell, out, res)
    # a capturing stream: refused before any CUDA work, the capture stays valid
    x = torch.zeros(4, device="cuda")
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    before = ctx.launches
    with torch.cuda.graph(g, stream=s):
        rc = lib.lz4b200_stream_decode_to_device_at_async(ctx.handle, src.data_ptr(), len(wire), cell.data_ptr(), 65536,
                                                          out.data_ptr(), len(data), res.data_ptr(),
                                                          torch.cuda.current_stream().cuda_stream)
        x.add_(1)
    assert rc == E_ARG and "capturing" in native.last_error() and ctx.launches == before
    g.replay()
    torch.cuda.synchronize()
    assert x.cpu().tolist() == [1.0] * 4
