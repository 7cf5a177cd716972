"""The asynchronous LZ4Stream calls on an H100: lz4b200_stream_encode_from_device_async (n bytes of device memory written
as one LZ4Stream into page-locked host memory) and lz4b200_stream_decode_to_device_async (a whole stream in page-locked
host memory decoded into device memory).

The encode's size and bytes must be those of lz4b200_stream_encode_from_device over many pipeline stages, at every chunk
size, in fast and HC mode, with out_size in device or page-locked memory; the decode must restore both the synchronous
call's streams and the asynchronous encode's, and report every status lz4b200_stream_decode_to_device reports -- from the
call where the host decides it, in out_size where the device does.  Both calls return while the device is busy, are
ordered on the caller's stream, and refuse the wrong kind of memory, bad arguments and a capturing stream."""
import functools

import numpy as np
import pytest

import oracle
from tests import cases
from tests.test_mixed_memory_gpu import _dev, _Options

pytestmark = pytest.mark.gpu

CLASSES = ("E0", "E50", "E100", "ETEXT", "MIX")
N = 3 * (1 << 20) + 12345                                    # not a multiple of any chunk size below
BLOCKS = (16, 4096, 65536, 1 << 20, N + 1)
CANARY = 0x5C
G = 64                                                       # canary bytes around a device output
E_ARG, E_FORMAT = -1, -5


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@functools.lru_cache(maxsize=None)
def _data(cls, n=N):
    if cls != "MIX":
        return cases.content(cls, n, seed=70).tobytes()
    parts = [cases.content(c, n // 4 + 1, seed=71 + i).tobytes() for i, c in enumerate(("E0", "E50", "E100", "ETEXT"))]
    return b"".join(parts)[:n]


def _pinned(n, fill, dtype=None):
    import torch
    return torch.full((n,), fill, dtype=dtype or torch.uint8).pin_memory()


def _pinned_bytes(buf):
    t = _pinned(max(len(buf), 1), 0)
    t.numpy()[:len(buf)] = np.frombuffer(buf, np.uint8)
    return t


def _size_cell(kind):
    """out_size (int64[1]) followed by a canary cell, in device memory or page-locked host memory."""
    import torch
    if kind == "device":
        return torch.full((2,), -7, dtype=torch.int64, device="cuda")
    return _pinned(2, -7, torch.int64)


def _bound(n, bs):
    from lz4net_b200 import native
    return int(native.lib().lz4b200_stream_bound(n, bs))


def _sync_encode(ctx, raw, bs, hc):
    from lz4net_b200 import batch
    return batch.stream_encode_to_host(ctx, raw, block_size=bs, hc=hc).tobytes()


def _async_encode(ctx, raw, bs, hc, kind, stream=None):
    """Returns (wire bytes, the size cell's two values, the bytes of dst behind the stream)."""
    import torch
    from lz4net_b200 import batch
    dst = _pinned(_bound(raw.numel(), bs) + G, CANARY)
    size = _size_cell(kind)
    batch.stream_encode_to_host_async(ctx, raw, dst[:dst.numel() - G], size, block_size=bs, hc=hc, stream=stream)
    torch.cuda.synchronize()
    w = int(size[0])
    return dst.numpy()[:max(w, 0)].tobytes(), size.cpu().tolist(), dst.numpy()[max(w, 0):]


# ---- encode -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bs", BLOCKS, ids=lambda b: f"bs{b}")
@pytest.mark.parametrize("hc", [False, True], ids=["fast", "hc"])
@pytest.mark.parametrize("cls", CLASSES)
def test_gpu_async_stream_encode_equals_the_synchronous_encode(ctx, cls, hc, bs):
    raw = _dev(np.frombuffer(_data(cls), np.uint8))
    want = _sync_encode(ctx, raw, bs, hc)
    with _Options(ctx, host_chunk_mb=1):                            # many stages, more than the two asynchronous slots
        for kind in ("device", "pinned"):
            got, size, behind = _async_encode(ctx, raw, bs, hc, kind)
            assert size == [len(want), -7], kind                        # the canary cell behind out_size is intact
            assert got == want, kind
            assert (behind == CANARY).all(), kind                       # nothing written behind the stream


def test_gpu_async_stream_encode_of_nothing_and_of_tiny_inputs(ctx):
    import torch
    for n in (0, 1, 15, 16, 17):
        raw = _dev(np.frombuffer(_data("ETEXT", 64)[:n], np.uint8)) if n else torch.zeros(0, dtype=torch.uint8, device="cuda")
        for hc in (False, True):
            want = _sync_encode(ctx, raw, 16, hc) if n else b""
            got, size, behind = _async_encode(ctx, raw, 16, hc, "pinned")
            assert size == [len(want), -7] and got == want and (behind == CANARY).all(), (n, hc)


# ---- decode -----------------------------------------------------------------------------------------------------------
def _async_decode(ctx, wire, n, cap, kind="device", stream=None):
    """Decodes the first n bytes of `wire` (bytes) into a device buffer of cap bytes with G canary bytes in front and behind.
    Returns (the call's status, the size cell, the decoded bytes of cap, the canaries in front and behind)."""
    import torch
    from lz4net_b200 import native
    src = _pinned_bytes(wire)
    out = torch.full((cap + 2 * G,), CANARY, dtype=torch.uint8, device="cuda")
    size = _size_cell(kind)
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = native.lib().lz4b200_stream_decode_to_device_async(ctx.handle, src.data_ptr(), n, out.data_ptr() + G, cap,
                                                            size.data_ptr(), st)
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    return rc, size.cpu().tolist(), o[G:G + cap].tobytes(), o[:G], o[G + cap:]


def _sync_decode(ctx, wire, cap):
    """(status or decoded size, bytes) of lz4b200_stream_decode_to_device."""
    import torch
    from lz4net_b200 import native
    src = np.frombuffer(wire, np.uint8).copy() if wire else np.zeros(1, np.uint8)
    out = torch.full((max(cap, 1),), CANARY, dtype=torch.uint8, device="cuda")
    r = native.lib().lz4b200_stream_decode_to_device(ctx.handle, src.ctypes.data, len(wire), out.data_ptr(), cap,
                                                     torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return int(r), out.cpu().numpy()[:max(r, 0)].tobytes()


@pytest.mark.parametrize("bs", (16, 65536, 1 << 20), ids=lambda b: f"bs{b}")
@pytest.mark.parametrize("cls", CLASSES)
def test_gpu_async_stream_decode_round_trip(ctx, cls, bs):
    """The synchronous encode's wire, and the asynchronous encode's (read after a synchronise), decoded into device memory
    with canaries on both sides, over many stages; out_size in device and page-locked memory."""
    data = _data(cls)
    raw = _dev(np.frombuffer(data, np.uint8))
    with _Options(ctx, host_chunk_mb=1):
        wires = [_sync_encode(ctx, raw, bs, False), _async_encode(ctx, raw, bs, True, "device")[0]]
        for wire in wires:
            for kind in ("device", "pinned"):
                rc, size, got, front, behind = _async_decode(ctx, wire, len(wire), len(data) + 100, kind)
                assert rc == 0 and size == [len(data), -7], kind
                assert got[:len(data)] == data, kind
                assert set(got[len(data):]) <= {CANARY} and (front == CANARY).all() and (behind == CANARY).all(), kind


def _varint(v):
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def _chunk(flags, raw, payload, clen=None):
    return _varint(flags) + _varint(raw) + (_varint(len(payload) if clen is None else clen) if flags & 1 else b"") + payload


def _good(ctx):
    """A real stream of several chunks, compressed and stored, and its data."""
    data = _data("MIX", 300_000)
    return _sync_encode(ctx, _dev(np.frombuffer(data, np.uint8)), 65536, False), data


def test_gpu_async_stream_decode_refuses_malformed_headers_before_any_device_work(ctx):
    """A truncated stream, a varint that runs off the end, compLen > rawLen and a multi-pass flag: E_FORMAT from the call,
    as from the synchronous call, with dst and out_size untouched."""
    wire, data = _good(ctx)
    payload = oracle.encode(b"abcd" * 40)[1]
    bad = {
        "truncated": wire[:-1],
        "truncated-header": wire + b"\x01",
        "bad-varint": _chunk(0, 4, b"abcd") + b"\x81",
        "complen-above-rawlen": _chunk(1, 4, b"abcde"),
        "multi-pass": _chunk(1 | 4, 160, payload),
    }
    for name, w in bad.items():
        assert _sync_decode(ctx, w, len(data) + 200)[0] == E_FORMAT, name
        rc, size, got, front, behind = _async_decode(ctx, w, len(w), len(data) + 200, "pinned")
        assert rc == E_FORMAT and size == [-7, -7], name
        assert set(got) == {CANARY} and (front == CANARY).all() and (behind == CANARY).all(), name


def test_gpu_async_stream_decode_refuses_a_destination_too_small(ctx):
    wire, data = _good(ctx)
    assert _sync_decode(ctx, wire, len(data) - 1)[0] == E_ARG
    rc, size, got, front, behind = _async_decode(ctx, wire, len(wire), len(data) - 1)
    assert rc == E_ARG and size == [-7, -7] and set(got) == {CANARY} and (behind == CANARY).all()


def _crafted_equal_length_block():
    """A chunk flagged compressed whose LZ4 payload is exactly as long as its data (33 bytes both): 16 literals, a match of 5
    at offset 16, then 12 literals."""
    lit, tail = b"ABCDEFGHIJKLMNOP", b"0123456789xy"
    data = lit + lit[:5] + tail
    block = bytes([0xF1, 1]) + lit + b"\x10\x00" + bytes([0xC0]) + tail
    assert len(block) == len(data) == 33
    return data, block


def _decoded_size(wire):
    from lz4net_b200 import native
    src = np.frombuffer(wire, np.uint8).copy()
    return int(native.lib().lz4b200_stream_decoded_size(src.ctypes.data, len(wire)))


def test_gpu_async_stream_decode_statuses_found_on_the_device(ctx):
    """A compressed payload that does not decode from exactly its compLen bytes: out_size == E_FORMAT where the synchronous
    call returns E_FORMAT, the decoded size where it does not; a compressed chunk with compLen == rawLen is handled as the
    synchronous call handles it; good chunks around a bad one change nothing."""
    wire, data = _good(ctx)
    eq_data, eq_block = _crafted_equal_length_block()
    streams = {
        "good": wire,
        "garbage-payload": _chunk(1, 100, b"\xf0"),
        "short-match": _chunk(1, 100, bytes([0x1F, 0x41, 0x01, 0x00])),
        "good-then-garbage": wire + _chunk(1, 100, b"\xf0") + wire,
        "equal-length-compressed": _chunk(1, len(eq_data), eq_block),
        "equal-length-garbage": _chunk(1, 33, bytes(range(33))),
        "stored-then-equal": _chunk(0, 5, b"hello") + _chunk(1, len(eq_data), eq_block),
    }
    rng = np.random.default_rng(5)
    for k in range(6):                                                 # corrupted bytes inside a real stream's payloads
        w = bytearray(wire)
        for p in rng.integers(len(w) // 4, len(w), 3):
            w[p] ^= 0xFF
        streams[f"corrupt-{k}"] = bytes(w)
    saw_format = saw_ok = False
    for name, w in streams.items():
        cap = 2 * len(data) + 400
        want, want_bytes = _sync_decode(ctx, w, cap)
        rc, size, got, front, behind = _async_decode(ctx, w, len(w), cap)
        if want == E_ARG or (want == E_FORMAT and rc == E_FORMAT):             # refused by the header walk, as before
            assert rc == want and size == [-7, -7], name
            continue
        assert rc == 0 and size == [want, -7], (name, want, size)
        saw_format |= want == E_FORMAT
        if want >= 0:
            saw_ok = True
            assert got[:want] == want_bytes, name
        # nothing written outside [dst, dst + decoded size), whatever the status
        assert set(got[_decoded_size(w):]) <= {CANARY} and (front == CANARY).all() and (behind == CANARY).all(), name
    assert saw_format and saw_ok


def test_gpu_async_stream_decode_of_nothing(ctx):
    """n == 0, and a stream of empty chunks: out_size == 0, nothing else written."""
    empties = _chunk(0, 0, b"") * 5 + _chunk(2, 0, b"")
    for w, n in ((b"", 0), (empties, len(empties))):
        for kind in ("device", "pinned"):
            rc, size, got, front, behind = _async_decode(ctx, w, n, 16, kind)
            assert rc == 0 and size == [0, -7] and set(got) == {CANARY}, (n, kind)
        assert _sync_decode(ctx, w, 16)[0] == 0


# ---- non-blocking, ordering --------------------------------------------------------------------------------------------
def test_gpu_async_stream_calls_return_while_the_stream_is_busy(ctx):
    import torch
    from lz4net_b200 import batch
    data = _data("MIX", 4 << 20)
    raw = _dev(np.frombuffer(data, np.uint8))
    wire = _sync_encode(ctx, raw, 65536, False)
    src = _pinned_bytes(wire)
    dst = _pinned(_bound(len(data), 65536), 0)
    out = torch.zeros(len(data), dtype=torch.uint8, device="cuda")
    size = _size_cell("device")
    s = torch.cuda.Stream()
    calls = {
        "encode": lambda: batch.stream_encode_to_host_async(ctx, raw, dst, size, block_size=65536, stream=s),
        "decode": lambda: batch.stream_decode_to_device_async(ctx, src, len(wire), out, size, stream=s),
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
                assert int(size[0]) == (len(wire) if name == "encode" else len(data)), name
    assert dst.numpy()[:len(wire)].tobytes() == wire
    assert out.cpu().numpy().tobytes() == data


def test_gpu_async_stream_calls_are_ordered_on_the_callers_stream_and_between_streams(ctx):
    """Per stream, with no host synchronisation: a sleep, a producer filling the device input, the asynchronous encode of
    it, the asynchronous decode of a stream written earlier, and consumers of both results; two streams, one context."""
    import torch
    from lz4net_b200 import batch, synth
    n, bs = 64, 65536
    want_raw = np.concatenate([synth.make_blocks(c, n // 4, bs, seed=9, first_block=k * (n // 4)).reshape(-1)
                               for k, c in enumerate(synth.CLASSES)])
    want = _sync_encode(ctx, _dev(want_raw), 1 << 16, False)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    raws = [torch.zeros(n * bs, dtype=torch.uint8, device="cuda") for _ in streams]
    dsts = [_pinned(_bound(n * bs, 1 << 16), 0xFF) for _ in streams]
    srcs = [_pinned_bytes(want) for _ in streams]
    backs = [torch.zeros(n * bs, dtype=torch.uint8, device="cuda") for _ in streams]
    got = []
    with _Options(ctx, host_chunk_mb=1):
        for s, raw, dst, src, back in zip(streams, raws, dsts, srcs, backs):
            with torch.cuda.stream(s):
                esize, dsize = _size_cell("device"), _size_cell("pinned")
                torch.cuda._sleep(50_000_000)
                for k, c in enumerate(synth.CLASSES):                  # the producer: enqueued, not yet run
                    batch.synth_fill(ctx, raw[k * (n // 4) * bs:], n // 4, bs, synth.CLASS_ID[c], seed=9, first_block=k * (n // 4))
                batch.stream_encode_to_host_async(ctx, raw, dst, esize, block_size=1 << 16)
                batch.stream_decode_to_device_async(ctx, src, len(want), back, dsize)
                got.append((esize.clone(), back.clone(), dsize))             # the consumers
        torch.cuda.synchronize()
    for dst, (esize, back, dsize) in zip(dsts, got):
        assert esize.cpu().tolist() == [len(want), -7] and dsize.tolist() == [n * bs, -7]
        assert dst.numpy()[:len(want)].tobytes() == want
        assert back.cpu().numpy().tobytes() == want_raw.tobytes()


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_gpu_async_stream_calls_refuse_wrong_memory_and_bad_arguments(ctx):
    import torch
    from lz4net_b200 import native
    lib = native.lib()
    data = _data("ETEXT", 8192)
    raw = _dev(np.frombuffer(data, np.uint8))
    wire = _sync_encode(ctx, raw, 4096, False)
    bound = _bound(len(data), 4096)
    pk_dst, pk_src = _pinned(bound, CANARY), _pinned_bytes(wire)
    out = torch.full((len(data),), CANARY, dtype=torch.uint8, device="cuda")
    dsize, psize, hsize = _size_cell("device"), _size_cell("pinned"), np.full(2, -7, np.int64)
    pageable, device = np.full(bound, CANARY, np.uint8), torch.full((bound,), CANARY, dtype=torch.uint8, device="cuda")
    pageable_wire = np.frombuffer(wire, np.uint8).copy()

    def enc(src=raw.data_ptr(), n=len(data), bs=4096, dst=pk_dst.data_ptr(), cap=bound, size=dsize.data_ptr()):
        return lib.lz4b200_stream_encode_from_device_async(ctx.handle, src, n, bs, 0, dst, cap, size, 0)

    def dec(src=pk_src.data_ptr(), n=len(wire), dst=out.data_ptr(), cap=len(data), size=psize.data_ptr()):
        return lib.lz4b200_stream_decode_to_device_async(ctx.handle, src, n, dst, cap, size, 0)

    refused = {
        "encode pageable dst": (lambda: enc(dst=pageable.ctypes.data), "dst must be page-locked"),
        "encode device dst": (lambda: enc(dst=device.data_ptr()), "dst must be page-locked"),
        "encode pageable src": (lambda: enc(src=pageable.ctypes.data), "src must be device memory"),
        "encode page-locked src": (lambda: enc(src=pk_src.data_ptr(), n=len(wire), cap=_bound(len(wire), 4096)), "src must be device memory"),
        "encode pageable out_size": (lambda: enc(size=hsize.ctypes.data), "out_size must be"),
        "encode n < 0": (lambda: enc(n=-1), "bad argument"),
        "encode block_size < 1": (lambda: enc(bs=0), "bad argument"),
        "encode block_size above a frame": (lambda: enc(bs=2**31 - 1), "a chunk's frame must fit an int32"),
        "encode dst_cap < bound": (lambda: enc(cap=bound - 1), "lz4b200_stream_bound"),
        "encode null out_size": (lambda: enc(size=None), "bad argument"),
        "decode pageable src": (lambda: dec(src=pageable_wire.ctypes.data), "src must be page-locked"),
        "decode device src": (lambda: dec(src=device.data_ptr()), "src must be page-locked"),
        "decode page-locked dst": (lambda: dec(dst=pk_dst.data_ptr()), "dst must be device memory"),
        "decode pageable dst": (lambda: dec(dst=pageable.ctypes.data), "dst must be device memory"),
        "decode pageable out_size": (lambda: dec(size=hsize.ctypes.data), "out_size must be"),
        "decode n < 0": (lambda: dec(n=-1), "bad argument"),
        "decode null out_size": (lambda: dec(size=None), "bad argument"),
    }
    before = ctx.launches
    for name, (call, text) in refused.items():
        assert call() == E_ARG, name
        assert text in native.last_error(), (name, native.last_error())
    assert ctx.launches == before                                       # nothing enqueued
    torch.cuda.synchronize()
    assert dsize.cpu().tolist() == [-7, -7] and psize.tolist() == [-7, -7] and hsize.tolist() == [-7, -7]
    assert (out.cpu().numpy() == CANARY).all() and (pk_dst.numpy() == CANARY).all()
    assert (pageable == CANARY).all() and (device.cpu().numpy() == CANARY).all()


def test_gpu_async_stream_refusal_texts(ctx):
    """Each refusal names what is wrong (checked one call at a time: the error text is the last call's)."""
    import torch
    from lz4net_b200 import native
    lib = native.lib()
    raw = _dev(np.frombuffer(_data("E50", 4096), np.uint8))
    bound = _bound(4096, 1024)
    pk = _pinned(bound, 0)
    pageable = np.zeros(bound, np.int64)
    size = _size_cell("device")
    assert lib.lz4b200_stream_encode_from_device_async(ctx.handle, raw.data_ptr(), 4096, 1024, 0, pageable.ctypes.data, bound,
                                                       size.data_ptr(), 0) == E_ARG
    assert "dst must be page-locked host memory" in native.last_error()
    assert lib.lz4b200_stream_encode_from_device_async(ctx.handle, raw.data_ptr(), 4096, 1024, 0, pk.data_ptr(), bound,
                                                       pageable.ctypes.data, 0) == E_ARG
    assert "out_size must be device memory of the context's GPU or page-locked host memory" in native.last_error()
    assert lib.lz4b200_stream_encode_from_device_async(ctx.handle, pk.data_ptr(), 4096, 1024, 0, pk.data_ptr(), bound,
                                                       size.data_ptr(), 0) == E_ARG
    assert "src must be device memory of the context's GPU" in native.last_error()
    assert lib.lz4b200_stream_decode_to_device_async(ctx.handle, pageable.ctypes.data, 16, raw.data_ptr(), 4096,
                                                     size.data_ptr(), 0) == E_ARG
    assert "src must be page-locked host memory" in native.last_error()
    torch.cuda.synchronize()
    assert size.cpu().tolist() == [-7, -7]


def test_gpu_async_stream_calls_refuse_a_capturing_stream_and_leave_the_capture_valid(ctx):
    import torch
    from lz4net_b200 import native
    lib = native.lib()
    data = _data("E50", 8192)
    raw = _dev(np.frombuffer(data, np.uint8))
    wire = _sync_encode(ctx, raw, 4096, True)
    dst, src = _pinned(_bound(len(data), 4096), 0), _pinned_bytes(wire)
    size = _size_cell("device")
    out = torch.zeros(len(data), dtype=torch.uint8, device="cuda")
    x = torch.zeros(4, device="cuda")
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    before = ctx.launches
    rcs = []
    with torch.cuda.graph(g, stream=s):
        st = torch.cuda.current_stream().cuda_stream
        rcs.append(lib.lz4b200_stream_encode_from_device_async(ctx.handle, raw.data_ptr(), len(data), 4096, 1, dst.data_ptr(),
                                                               dst.numel(), size.data_ptr(), st))
        rcs.append(lib.lz4b200_stream_decode_to_device_async(ctx.handle, src.data_ptr(), len(wire), out.data_ptr(), out.numel(),
                                                             size.data_ptr(), st))
        x.add_(1)
    assert rcs == [E_ARG] * 2 and "capturing" in native.last_error()
    assert ctx.launches == before
    g.replay()
    torch.cuda.synchronize()
    assert x.cpu().tolist() == [1.0] * 4
    assert size.cpu().tolist() == [-7, -7]
