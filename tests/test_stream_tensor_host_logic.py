"""LZ4Stream.Write(tensor) / ReadInto(tensor) without a GPU: the class reaches the device through its context
(stream_encode_from_device / stream_decode_to_device), so a stand-in context built on the oracle, taking CPU tensors in
place of device memory, covers the chunk-boundary logic: mixed host and tensor writes give the wire bytes of host-only
writes, whole blocks go through the device call, and ReadInto keeps Read's semantics, InteractiveRead included.  The GPU
twin is tests/test_stream_mixed_gpu.py."""
import io

import numpy as np
import pytest
import torch

from lz4net_b200 import codec
from tests import cases
from tests.test_stream_host_logic import OracleContext, _chunk_ends

S, M, F = codec.LZ4Stream, codec.LZ4StreamMode, codec.LZ4StreamFlags
BS = 4096


class TensorOracleContext(OracleContext):
    """The oracle stand-in plus the two device calls, on CPU tensors; records what went through them."""

    def __init__(self):
        self.encoded, self.decoded = [], []

    def stream_encode_from_device(self, t, bs, hc):
        assert t.dtype == torch.uint8 and t.dim() == 1 and t.numel() % bs == 0    # whole blocks only
        self.encoded.append(t.numel())
        return self.stream_encode(t.numpy().tobytes(), bs, hc)

    def stream_decode_to_device(self, raw, out):
        d = self.stream_decode(raw)
        assert len(d) <= out.numel()
        out[:len(d)] = torch.frombuffer(bytearray(d), dtype=torch.uint8) if d else out[:0]
        self.decoded.append(len(d))
        return len(d)


@pytest.fixture(scope="module")
def data():
    return (cases.content("ETEXT", 7 * BS + 33, seed=3).tobytes() + cases.content("E0", 3 * BS, seed=3).tobytes()
            + cases.content("E100", BS + 100, seed=3).tobytes())


def _host_wire(ctx, data, ops, hc):
    out = io.BytesIO()
    with S(out, M.Compress, F.IsolateInnerStream | (F.HighCompression if hc else 0), BS, batchBlocks=3, context=ctx) as w:
        for kind, a, b in ops:
            if kind == "flush":
                w.Flush()
            else:
                w.Write(data, a, b - a)
    return out.getvalue()


@pytest.mark.parametrize("hc", [False, True])
@pytest.mark.parametrize("seed", range(6))
def test_mixed_tensor_and_host_writes_equal_host_writes(data, hc, seed):
    """Random cuts, each written from host memory or from a tensor (int32 ones too: their bytes in storage order),
    random Flushes: the wire equals the same writes all from host memory, and whole blocks went through the device."""
    rng = np.random.default_rng(seed)
    ops, pos = [], 0
    while pos < len(data):
        k = int(min(len(data) - pos, rng.choice([1, 7, BS - 1, BS, BS + 1, 3 * BS + 5, int(rng.integers(1, 5 * BS))])))
        ops.append(("tensor" if rng.integers(0, 2) else "host", pos, pos + k)); pos += k
        if rng.integers(0, 4) == 0:
            ops.append(("flush", 0, 0))
    ctx = TensorOracleContext()
    want = _host_wire(ctx, data, ops, hc)
    out = io.BytesIO()
    with S(out, M.Compress, F.IsolateInnerStream | (F.HighCompression if hc else 0), BS, batchBlocks=3, context=ctx) as w:
        for kind, a, b in ops:
            if kind == "flush":
                w.Flush()
            elif kind == "host":
                w.Write(data[a:b])
            elif (b - a) % 4 == 0 and a % 2:
                w.Write(torch.frombuffer(bytearray(data[a:b]), dtype=torch.int32))
            else:
                big = torch.frombuffer(bytearray(b"\0" * 5 + data[a:b] + b"\0" * 3), dtype=torch.uint8)
                w.Write(big, 5, b - a)                                              # an offset and a count into it
    assert out.getvalue() == want
    assert _chunk_ends(want) and all(n % BS == 0 for n in ctx.encoded)


def test_tensor_write_sends_whole_blocks_to_the_device(data):
    """A pending partial chunk is completed from the tensor's head (less than a block crosses to the host), the whole
    blocks are encoded from the tensor, the tail stays pending until Flush."""
    ctx = TensorOracleContext()
    out = io.BytesIO()
    w = S(out, M.Compress, F.IsolateInnerStream, BS, context=ctx)
    w.Write(data[:100])
    t = torch.frombuffer(bytearray(data[100:100 + 5 * BS + 7]), dtype=torch.uint8)
    w.Write(t)
    assert ctx.encoded == [4 * BS] and len(w._pending) == 7 + 100                   # head BS - 100, 4 blocks, tail
    w.Close()
    assert out.getvalue() == ctx.stream_encode(data[:100 + 5 * BS + 7], BS, False)
    with pytest.raises(ValueError):
        S(io.BytesIO(), M.Compress, context=ctx).Write(t, 10, t.numel())


@pytest.fixture(scope="module")
def stream(data):
    ctx = TensorOracleContext()
    wire = ctx.stream_encode(data, BS, False) + ctx.stream_encode(data[:BS + 9], BS, False)   # two streams back to back
    whole = data + data[:BS + 9]
    sizes = [min(BS, len(data) - o) for o in range(0, len(data), BS)] + [BS, 9]
    return wire, whole, _chunk_ends(wire), sizes


def test_interactive_read_into_takes_one_chunk_at_a_time(stream):
    wire, whole, ends, sizes = stream
    ctx = TensorOracleContext()
    inner = io.BytesIO(wire)
    r = S(inner, M.Decompress, F.InteractiveRead, batchBlocks=256, context=ctx)
    back = bytearray()
    out = torch.zeros(3 * BS, dtype=torch.uint8)
    for k in range(len(ends)):
        n = r.ReadInto(out)
        assert inner.tell() == ends[k] and n == sizes[k]                            # one chunk read, one chunk returned
        back += out[:n].numpy().tobytes()
    assert r.ReadInto(out) == 0 and bytes(back) == whole
    assert ctx.decoded and all(d <= BS for d in ctx.decoded)                         # decoded straight into the tensor


def test_read_into_straddling_chunk_and_mixed_reads(stream):
    """Non-interactive: a tensor whose end falls inside a chunk gets the whole chunks before it directly and the rest of
    that chunk through the host; what is left of it comes first in the next Read or ReadInto."""
    wire, whole, _, _ = stream
    ctx = TensorOracleContext()
    r = S(io.BytesIO(wire), M.Decompress, batchBlocks=4, context=ctx)
    a = torch.zeros(2 * BS + 10, dtype=torch.uint8)
    assert r.ReadInto(a) == a.numel() and a.numpy().tobytes() == whole[:a.numel()]
    assert ctx.decoded == [2 * BS]                                                  # two whole chunks straight in
    got = bytearray(r.Read(5))
    rest = torch.zeros(len(whole), dtype=torch.int16)                               # any dtype: its bytes
    n = r.ReadInto(rest)
    assert n == len(whole) - a.numel() - 5
    got += rest.numpy().tobytes()[:n]
    assert a.numpy().tobytes() + bytes(got) == whole and r.ReadInto(rest) == 0 and r.Read(3) == b""
    with pytest.raises(NotImplementedError):
        S(io.BytesIO(), M.Compress, context=ctx).ReadInto(a)


def test_read_into_truncated_stream(stream):
    wire, whole, _, _ = stream
    with pytest.raises(EOFError):
        S(io.BytesIO(wire[:-2]), M.Decompress, context=TensorOracleContext()).ReadInto(torch.zeros(len(whole) + 1, dtype=torch.uint8))
