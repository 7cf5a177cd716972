"""LZ4Stream between device and host memory on an H100: lz4b200_stream_encode_from_device (raw bytes in HBM, wire bytes
to host memory) and lz4b200_stream_decode_to_device (wire bytes in host memory, decoded into HBM).

The wire bytes must equal lz4b200_stream_encode of a host copy and the oracle-built reference stream; the decode must give
back the raw bytes, write nothing outside [dst, dst + decoded size), and report the statuses of lz4b200_stream_decode;
both calls are ordered behind the work already queued on the caller's stream and refuse the wrong kind of memory."""
import functools
import io

import numpy as np
import pytest

import oracle
from tests import cases
from tests.test_gpu_parity import _ref_stream
from tests.test_mixed_memory_gpu import _busy, _host, _Options, CHUNK_MB_DEFAULT
from tests.test_stream_host_logic import _chunk_ends, _varint

pytestmark = pytest.mark.gpu

E_ARG, E_FORMAT = -1, -5
DEV_GUARD, HOST_GUARD = 0xA5, 0xEE
BLOCKS = (16, 1000, 65536, 65547, 1 << 20)


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


def _lengths(bs):
    return [0, 1, bs - 1, bs, bs + 1, 3 * bs + (bs // 3 if bs < (1 << 20) else 12345)]


def _dev(data, skew=3):
    """The bytes on the device, `skew` bytes into their allocation (a misaligned source)."""
    import torch
    t = torch.zeros(len(data) + skew + 16, dtype=torch.uint8, device="cuda")
    if data:
        t[skew:skew + len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    return t[skew:skew + len(data)]


def _encode(ctx, t, n, bs, hc, dst):
    from lz4net_b200 import native
    return native.lib().lz4b200_stream_encode_from_device(ctx.handle, t.data_ptr(), n, bs, int(hc), dst.ctypes.data,
                                                          dst.nbytes, 0)


@functools.lru_cache(maxsize=None)
def _ref(data, bs, hc):
    return _ref_stream(data, bs, hc)


@pytest.mark.parametrize("pinned,chunk_mb", [(False, CHUNK_MB_DEFAULT), (True, 1), (True, CHUNK_MB_DEFAULT)],
                         ids=["pageable-default-stages", "pinned-many-stages", "pinned-default-stages"])
@pytest.mark.parametrize("mode", ["fast", "hc-auto", "hc0", "hc1", "hc2"])
def test_gpu_stream_encode_from_device_equals_host_and_reference(ctx, mode, pinned, chunk_mb):
    """Block sizes 16 .. 1 MiB, lengths 0, 1, block - 1, block, block + 1 and several blocks, every content model in turn,
    a misaligned device source, host guard bytes behind the stream.  (The thread-per-block HC kernel, hc0, skips the
    1 MiB blocks: one thread encoding a MiB takes seconds.)"""
    from lz4net_b200 import native
    hc = mode != "fast"
    opts = {"host_chunk_mb": chunk_mb}
    if mode in ("hc0", "hc1", "hc2"):
        opts["hc_kernel"] = int(mode[2])
    k = 0
    with _Options(ctx, **opts):
        for bs in BLOCKS if mode != "hc0" else BLOCKS[:-1]:
            for n in _lengths(bs):
                data = cases.content(cases.MODELS[k % len(cases.MODELS)], n, seed=100 + k).tobytes()
                k += 1
                bound = int(native.lib().lz4b200_stream_bound(n, bs))
                dst = _host(bound + 64, HOST_GUARD, pinned)
                w = _encode(ctx, _dev(data), n, bs, hc, dst[:bound])
                want = ctx.stream_encode(data, bs, hc)
                assert w == len(want) and dst[:w].tobytes() == want, (mode, bs, n)
                assert (dst[w:] == HOST_GUARD).all(), (mode, bs, n)
                if not hc or n <= 300000 or chunk_mb == 1:
                    assert want == _ref(data, bs, hc), (mode, bs, n)
                if n:
                    assert _encode(ctx, _dev(data), n, bs, hc, dst[:bound - 1]) == E_ARG       # one byte short


def _decode(ctx, wire, cap, guard=37):
    """Decodes host bytes `wire` into a device buffer of `cap` bytes with `guard` guard bytes on both sides.  Returns
    (status, the cap bytes, whether the guards are intact); the host form's status for comparison."""
    import torch
    from lz4net_b200 import native
    src = np.frombuffer(bytes(wire) + b"\0", np.uint8)
    big = torch.full((cap + 2 * guard,), DEV_GUARD, dtype=torch.uint8, device="cuda")
    r = native.lib().lz4b200_stream_decode_to_device(ctx.handle, src.ctypes.data, len(wire), big.data_ptr() + guard, cap, 0)
    h = big.cpu().numpy()
    host = np.zeros(max(cap, 1), np.uint8)
    want = native.lib().lz4b200_stream_decode(ctx.handle, src.ctypes.data, len(wire), host.ctypes.data, cap)
    return r, want, h[guard:guard + cap], (h[:guard] == DEV_GUARD).all() and (h[guard + cap:] == DEV_GUARD).all()


def _cases(ctx):
    """(wire, raw): streams from either encoder, fast and HC, with stored, zero-length and HC-flagged chunks, streams
    back to back with partial chunks, and a compressed chunk whose compLen equals its rawLen."""
    from lz4net_b200 import batch
    out = []
    for i, (m, n, bs) in enumerate((("ETEXT", 300000, 65536), ("E100", 200000, 65536), ("E0", 70000, 1000),
                                    ("mixed", 1 << 21, 1 << 20), ("E50", 5000, 16), ("lowent", 65547 * 2 + 5, 65547))):
        d = cases.content(m, n, seed=40 + i).tobytes()
        for hc in (False, True):
            out.append((ctx.stream_encode(d, bs, hc), d))
            out.append((batch.stream_encode_to_host(ctx, _dev(d), bs, hc).tobytes(), d))
    a, b = cases.content("ETEXT", 100000, seed=1).tobytes(), cases.content("E100", 7000, seed=2).tobytes()
    empty = _varint(0) + _varint(0)                                             # a zero-length stored chunk
    empty_c = _varint(3) + _varint(0) + _varint(0)                              # a zero-length compressed HC chunk
    out.append((ctx.stream_encode(a, 65536, True) + empty + ctx.stream_encode(b, 4096, False) + empty_c, a + b))
    lit, last = b"abcdefgh", b"0123456789ABCD"
    blk = bytes([8 << 4]) + lit + bytes([4, 0, 14 << 4]) + last                 # 26 bytes that decode to 26 bytes
    raw = lit + b"efgh" + last
    assert oracle.decode_known(blk, len(raw)) == (len(blk), raw)
    out.append((_varint(1) + _varint(len(raw)) + _varint(len(blk)) + blk + ctx.stream_encode(a[:5000], 1000, False), raw + a[:5000]))
    return out


@pytest.mark.parametrize("chunk_mb", [1, CHUNK_MB_DEFAULT], ids=["many-stages", "default-stages"])
def test_gpu_stream_decode_to_device_round_trip(ctx, chunk_mb):
    from lz4net_b200 import batch
    with _Options(ctx, host_chunk_mb=chunk_mb):
        for wire, raw in _cases(ctx):
            r, want, h, guards = _decode(ctx, wire, len(raw) + 100)
            assert r == want == len(raw) and h[:len(raw)].tobytes() == raw
            assert guards and (h[len(raw):] == DEV_GUARD).all(), "a byte outside [dst, dst + decoded size) changed"
            out = _dev(b"\0" * len(raw), 0)
            pinned = _host(len(wire), 0, True)
            pinned[:] = np.frombuffer(wire, np.uint8)
            assert batch.stream_decode_to_device(ctx, pinned, out) == len(raw)
            assert out.cpu().numpy().tobytes() == raw


def test_gpu_stream_decode_statuses_equal_the_host_form(ctx):
    """Truncated streams and corrupt headers (nothing written), corrupt payloads, a capacity one byte short, n = 0."""
    d = cases.content("ETEXT", 200000, seed=5).tobytes() + cases.content("E100", 70000, seed=5).tobytes()
    wire = ctx.stream_encode(d, 65536, False)
    ends = _chunk_ends(wire)
    bad = [wire[:k] for k in (1, 2, 3, ends[0] - 1, ends[0] + 1, ends[0] + 3, len(wire) - 1)]   # truncated
    bad += [wire[:ends[0]] + b for b in (                                        # a valid chunk, then a corrupt header
        _varint(1) + _varint(10) + _varint(11) + bytes(11),                      # compLen > rawLen
        _varint(0) + _varint(1 << 31),                                           # a length no int holds
        _varint(5) + _varint(10) + _varint(5) + bytes(5),                        # compressed multi-pass chunk
        _varint(0) + _varint(100) + bytes(99))]                                  # payload cut short
    for b in bad:
        r, want, h, guards = _decode(ctx, b, len(d) + 10)
        assert r == want == E_FORMAT and guards and (h == DEV_GUARD).all(), len(b)
    n_fmt = 0
    for k in range(12):
        c = bytearray(wire)
        p = ends[k % 3] + 7 + 97 * k                                             # inside a compressed payload
        c[p] ^= 0x5A + k
        r, want, _, guards = _decode(ctx, bytes(c), len(d))
        assert r == want and guards, k
        n_fmt += r == E_FORMAT
    assert n_fmt > 0
    r, want, h, guards = _decode(ctx, wire, len(d) - 1)
    assert r == want == E_ARG and guards and (h == DEV_GUARD).all()
    r, want, h, guards = _decode(ctx, wire, len(d))
    assert r == want == len(d) and h.tobytes() == d and guards
    assert _decode(ctx, b"", 0)[:2] == (0, 0)


def test_gpu_stream_calls_refuse_the_wrong_kind_of_memory(ctx):
    import torch
    from lz4net_b200 import native
    l = native.lib()
    d = cases.content("E50", 10000, seed=3).tobytes()
    wire = ctx.stream_encode(d, 4096, False)
    h_src, h_dst = np.frombuffer(d, np.uint8).copy(), np.zeros(20000, np.uint8)
    d_src, d_dst = _dev(d, 0), torch.zeros(20000, dtype=torch.uint8, device="cuda")
    h_wire, d_wire = np.frombuffer(wire, np.uint8).copy(), _dev(wire, 0)
    enc = l.lz4b200_stream_encode_from_device
    dec = l.lz4b200_stream_decode_to_device
    assert enc(ctx.handle, h_src.ctypes.data, len(d), 4096, 0, h_dst.ctypes.data, len(h_dst), 0) == E_ARG
    assert enc(ctx.handle, d_src.data_ptr(), len(d), 4096, 0, d_dst.data_ptr(), len(h_dst), 0) == E_ARG
    assert dec(ctx.handle, d_wire.data_ptr(), len(wire), d_dst.data_ptr(), 20000, 0) == E_ARG
    assert dec(ctx.handle, h_wire.ctypes.data, len(wire), h_dst.ctypes.data, 20000, 0) == E_ARG
    assert enc(ctx.handle, d_src.data_ptr(), len(d), 2 ** 31 - 11, 0, h_dst.ctypes.data, len(h_dst), 0) == E_ARG
    assert enc(ctx.handle, d_src.data_ptr(), len(d), 0, 0, h_dst.ctypes.data, len(h_dst), 0) == E_ARG
    assert enc(ctx.handle, d_src.data_ptr(), 0, 4096, 0, h_dst.ctypes.data, 0, 0) == 0
    assert enc(ctx.handle, d_src.data_ptr(), len(d), 4096, 0, h_dst.ctypes.data, len(h_dst), 0) == len(wire)   # the right sides
    assert dec(ctx.handle, h_wire.ctypes.data, len(wire), d_dst.data_ptr(), 20000, 0) == len(d)
    assert d_dst[:len(d)].cpu().numpy().tobytes() == d


def test_gpu_stream_encode_waits_for_the_producer_on_its_stream(ctx):
    """synth_fill queued on a non-default stream behind a long kernel chain, then at once an encode given that stream:
    the encode reads the filled data, the same as after a synchronise."""
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 256, 65536

    def run(sync):
        raw = torch.zeros(nb * bs, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        _busy(s)
        with torch.cuda.stream(s):
            batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID["E50"], seed=7)
            if sync:
                s.synchronize()
            return batch.stream_encode_to_host(ctx, raw, bs).tobytes(), raw

    w0, _ = run(False)
    w1, raw = run(True)
    assert w0 == w1 and len(w1) < nb * bs * 0.9                                  # E50 data, not zeros
    assert w1 == ctx.stream_encode(raw.cpu().numpy().tobytes(), bs, False)


@pytest.mark.parametrize("hc", [False, True])
def test_gpu_lz4stream_tensor_write_and_read_into(ctx, hc):
    """LZ4Stream.Write of CUDA tensors mixed with host writes and Flushes gives the host-only wire bytes; ReadInto a CUDA
    tensor, plain and InteractiveRead, gives back the data."""
    import torch
    from lz4net_b200 import LZ4Stream, LZ4StreamFlags, LZ4StreamMode
    rng = np.random.default_rng(8)
    bs = 65536
    data = b"".join(cases.content(m, n, seed=6).tobytes() for m, n in (("ETEXT", 400000), ("E100", 150000), ("mixed", 90001)))
    flags = LZ4StreamFlags.IsolateInnerStream | (LZ4StreamFlags.HighCompression if hc else 0)
    cuts, pos, host = [0], 0, io.BytesIO()
    tw = io.BytesIO()
    with LZ4Stream(host, LZ4StreamMode.Compress, flags, bs, batchBlocks=4, context=ctx) as a, \
            LZ4Stream(tw, LZ4StreamMode.Compress, flags, bs, batchBlocks=4, context=ctx) as b:
        while pos < len(data):
            k = int(min(len(data) - pos, rng.integers(1, 3 * bs)))
            a.Write(data, pos, k)
            if rng.integers(0, 2):
                b.Write(_dev(data[pos:pos + k]))
            else:
                b.Write(data[pos:pos + k])
            pos += k
            if rng.integers(0, 5) == 0:
                a.Flush(); b.Flush()
    assert tw.getvalue() == host.getvalue()
    for interactive in (False, True):
        r = LZ4Stream(io.BytesIO(tw.getvalue()), LZ4StreamMode.Decompress,
                      LZ4StreamFlags.InteractiveRead if interactive else LZ4StreamFlags.Default, batchBlocks=3, context=ctx)
        back = bytearray()
        while True:
            out = torch.zeros(int(rng.integers(1, 3 * bs)), dtype=torch.uint8, device="cuda")
            n = r.ReadInto(out)
            if not n:
                break
            assert n <= bs or not interactive
            back += out[:n].cpu().numpy().tobytes()
        assert bytes(back) == data
