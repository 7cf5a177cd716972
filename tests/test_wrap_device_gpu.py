"""Wrap / Unwrap packets in device memory (lz4b200_wrap_batch_device, unwrap_batch_device, unwrap_batch_packed) on an H100.

Packets must be byte for byte those of the host lz4b200_wrap_batch and of LZ4Codec.Wrap's rule; statuses must be those of
the host lz4b200_unwrap_batch; nothing may be written outside a packet's bytes (wrap) or its output slot (unwrap); and the
calls must only enqueue work on the caller's stream."""
import hashlib
import struct

import numpy as np
import pytest

import oracle
from tests import cases

pytestmark = pytest.mark.gpu

LENS = (0, 1, 12, 13, 300, 65536, 65546, 65547, 70000, 1 << 20)
GUARD = 0xA5
E_ARG, E_FORMAT = -1, -5


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


def ref_wrap(d, hc):
    """LZ4Codec.Wrap / WrapHC (src/LZ4/LZ4Codec.cs:510-543) over the oracle encoders."""
    if not d:
        return bytes(8)
    r, o = (oracle.encode_hc if hc else oracle.encode)(d, cap=len(d))
    if r >= len(d) or r <= 0:
        return len(d).to_bytes(4, "little") * 2 + d
    return len(d).to_bytes(4, "little") + r.to_bytes(4, "little") + o


def _layout(sizes, skew, gap):
    """int64 offsets of `sizes` laid out with `gap` bytes between them, the first `skew` bytes in (misaligned)."""
    sizes = np.maximum(np.asarray(sizes, np.int64), 0)
    off = np.concatenate([[0], np.cumsum(sizes + gap)[:-1]]) + skew
    return off.astype(np.int64), int(off[-1] + sizes[-1] + gap) if len(sizes) else gap


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _src(blocks, skew=3, gap=5):
    so, total = _layout([len(b) for b in blocks], skew, gap)
    buf = np.zeros(total + 16, np.uint8)
    for o, b in zip(so, blocks):
        buf[o:o + len(b)] = np.frombuffer(b, np.uint8)
    return buf, so, np.array([len(b) for b in blocks], np.int32)


def _host_wrap(ctx, inputs, hc):
    from lz4net_b200 import native
    buf, so, sl = _src(inputs)
    caps = sl + 8
    do, total = _layout(caps, 0, 0)
    dst = np.zeros(total + 16, np.uint8)
    out = np.zeros(len(inputs), np.int32)
    native.check(native.lib().lz4b200_wrap_batch(ctx.handle, buf.ctypes.data, so.ctypes.data, sl.ctypes.data, int(hc), dst.ctypes.data,
                                                 do.ctypes.data, caps.ctypes.data, out.ctypes.data, len(inputs)), "wrap_batch")
    return [dst[o:o + r].tobytes() for o, r in zip(do, out)]


def _host_unwrap(ctx, packets, caps):
    from lz4net_b200 import native
    buf, so, sl = _src(packets)
    caps = np.asarray(caps, np.int32)
    do, total = _layout(caps, 0, 0)
    dst = np.zeros(total + 16, np.uint8)
    out = np.zeros(len(packets), np.int32)
    native.check(native.lib().lz4b200_unwrap_batch(ctx.handle, buf.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.ctypes.data,
                                                   do.ctypes.data, caps.ctypes.data, out.ctypes.data, len(packets)), "unwrap_batch")
    return out.tolist(), [dst[o:o + max(r, 0)].tobytes() for o, r in zip(do, out)]


def _device_wrap(ctx, inputs, hc, extra=()):
    """Inputs at misaligned offsets, packets in guard-filled slots at misaligned offsets with 0-2 spare bytes each.
    extra: (len, cap) of invalid packets appended (len < 0: no input).  Returns (out_len, packet bytes, host dst, do, caps)."""
    import torch
    from lz4net_b200 import batch
    blocks = list(inputs) + [b"\0" * max(l, 0) for l, _ in extra]
    buf, so, sl = _src(blocks)
    for i, (l, _) in enumerate(extra):
        sl[len(inputs) + i] = l
    caps = np.array([len(b) + 8 + i % 3 for i, b in enumerate(inputs)] + [c for _, c in extra], np.int32)
    do, total = _layout(caps, 7, 9)
    dst = torch.full((total + 64,), GUARD, dtype=torch.uint8, device="cuda")
    out = torch.full((len(blocks),), 12345, dtype=torch.int32, device="cuda")
    batch.wrap(ctx, _dev(buf), _dev(so), _dev(sl), dst, _dev(do), _dev(caps), out, hc=hc)
    torch.cuda.synchronize()
    res, h = out.cpu().tolist(), dst.cpu().numpy()
    return res, [h[o:o + max(r, 0)].tobytes() for o, r in zip(do, res)], h, do, caps


def _inputs():
    return [cases.content(m, n, seed=40 + i).tobytes() for i, m in enumerate(cases.MODELS) for n in LENS]


@pytest.mark.parametrize("mode", ["fast", "hc-auto", "hc0", "hc1", "hc2"])
def test_gpu_wrap_equals_host_and_reference(ctx, mode):
    inputs = _inputs()
    hc = mode != "fast"
    if mode in ("hc0", "hc1", "hc2"):
        ctx.set_option("hc_kernel", int(mode[2]))
    try:
        extra = [(100, 107), (0, 7), (-1, 100), (-5, 0)]                                     # capacity short by one, negative length
        res, pk, h, do, caps = _device_wrap(ctx, inputs, hc, extra)
    finally:
        ctx.set_option("hc_kernel", -1)
    host = _host_wrap(ctx, inputs, hc)
    n = len(inputs)
    for i, d in enumerate(inputs):
        assert pk[i] == host[i], (mode, i, len(d))
        if len(d) <= 70000 or i % 3 == 0:                                                   # (the oracle's HC on 1 MiB is slow)
            assert pk[i] == ref_wrap(d, hc), (mode, i, len(d))
    assert res[n:] == [E_ARG] * len(extra)
    written = np.zeros(len(h), bool)
    for o, r in zip(do, res):
        written[o:o + max(r, 0)] = True
    assert (h[~written] == GUARD).all(), "a byte outside [dst_off, dst_off + out_len) changed"
    assert sum(len(p) < len(d) + 8 for p, d in zip(pk, inputs)) > 10 and sum(len(p) == len(d) + 8 for p, d in zip(pk, inputs)) > 10


def _device_unwrap(ctx, packets, caps):
    import torch
    from lz4net_b200 import batch
    buf, so, sl = _src(packets, skew=5, gap=3)
    caps = np.asarray(caps, np.int32)
    do, total = _layout(caps, 11, 13)
    dst = torch.full((total + 64,), GUARD, dtype=torch.uint8, device="cuda")
    out = torch.full((len(packets),), 12345, dtype=torch.int32, device="cuda")
    batch.unwrap(ctx, _dev(buf), _dev(so), _dev(sl), dst, _dev(do), _dev(caps), out)
    torch.cuda.synchronize()
    res, h = out.cpu().tolist(), dst.cpu().numpy()
    slot = np.zeros(len(h), bool)
    for o, c in zip(do, caps):
        slot[o:o + max(c, 0)] = True
    assert (h[~slot] == GUARD).all(), "a byte outside [dst_off, dst_off + dst_cap) changed"
    return res, [h[o:o + max(r, 0)].tobytes() for o, r in zip(do, res)]


def _unwrap_packed(ctx, packets, room):
    import torch
    from lz4net_b200 import batch
    buf, so, sl = _src(packets, skew=1, gap=2)
    n = len(packets)
    dst = torch.full((max(room, 0) + 64,), GUARD, dtype=torch.uint8, device="cuda")
    out_off = torch.full((n + 1,), -7, dtype=torch.int64, device="cuda")
    out = torch.full((n,), 12345, dtype=torch.int32, device="cuda")
    batch.unwrap_packed(ctx, _dev(buf), _dev(so), _dev(sl), dst[:room], out_off, out)
    torch.cuda.synchronize()
    return out.cpu().tolist(), out_off.cpu().numpy(), dst.cpu().numpy()


@pytest.mark.parametrize("hc", [False, True])
def test_gpu_unwrap_round_trips(ctx, hc):
    inputs = _inputs()
    packets = _host_wrap(ctx, inputs, hc)
    res, outs = _device_unwrap(ctx, packets, [len(d) for d in inputs])
    assert res == [len(d) for d in inputs] and outs == inputs
    need = sum(len(d) for d in inputs)
    res, off, h = _unwrap_packed(ctx, packets, need)
    assert res == [len(d) for d in inputs] and off[0] == 0 and int(off[-1]) == need
    assert all(h[off[i]:off[i + 1]].tobytes() == d for i, d in enumerate(inputs))
    assert (h[need:] == GUARD).all()


def _corrupt(ctx):
    """(packet, capacity) pairs: every way lz4b200_unwrap_batch rejects a packet, next to good ones."""
    rng = np.random.default_rng(23)
    good = [cases.content(m, n, seed=n + i).tobytes() for i, m in enumerate(cases.MODELS) for n in (0, 13, 300, 5000, 65536)]
    pk = _host_wrap(ctx, good, False)
    out = []
    for d, p in zip(good, pk):
        raw, stored = struct.unpack("<ii", p[:8])
        size = max(raw, stored)
        out.append((p, size))                                                                 # good
        out.append((p, size - 1))                                                             # capacity one byte short
        out.append((p[:int(rng.integers(0, 8))], size))                                       # shorter than a header
        out.append((p[:8] + p[8:-1] if len(p) > 8 else p[:7], size))                          # stored > len - 8
        out.append((struct.pack("<iI", raw, 0x80000000 | stored) + p[8:], size))             # negative stored
        out.append((struct.pack("<Ii", 0x80000000 | raw, stored) + p[8:], size))             # negative raw
        out.append((p + b"\x00\x07", size))                                                   # trailing bytes after the payload
        if stored < raw:
            out.append((p[:8] + p[8:] + b"\x00", size))
            q = struct.pack("<ii", raw, stored + 1) + p[8:] + b"\x00"                         # read != stored (trailing byte counted)
            out.append((q, size))
            for k in range(4):                                                                # bit-flipped payloads
                b = bytearray(p)
                b[8 + int(rng.integers(0, stored))] ^= 1 << int(rng.integers(0, 8))
                out.append((bytes(b), size))
    return out


def test_gpu_unwrap_statuses_equal_host(ctx):
    pairs = _corrupt(ctx)
    packets, caps = [p for p, _ in pairs], [c for _, c in pairs]
    want, wout = _host_unwrap(ctx, packets, caps)
    got, gout = _device_unwrap(ctx, packets, caps)
    assert got == want
    for i, (w, a, b) in enumerate(zip(want, wout, gout)):
        if w >= 0:
            assert a == b, i
    assert {E_ARG, E_FORMAT} <= set(want) and sum(w >= 0 for w in want) > 20
    # the packed form: the sizes from the headers, the statuses of the host call at an unlimited capacity
    want_nolimit, wout = _host_unwrap_sized(ctx, packets)
    need = sum(max(s, 0) for s in _sizes(packets))
    res, off, h = _unwrap_packed(ctx, packets, need)
    assert res == want_nolimit
    assert list(np.diff(off)) == [max(s, 0) for s in _sizes(packets)]
    for i, (w, o) in enumerate(zip(want_nolimit, wout)):
        if w >= 0:
            assert h[off[i]:off[i] + w].tobytes() == o, i


def _sizes(packets):
    from lz4net_b200 import native
    l = native.lib()
    out = []
    for p in packets:
        b = np.frombuffer(p + b"\0", np.uint8)
        out.append(l.lz4b200_unwrap_size(b.ctypes.data, len(p)))
    return out


def _host_unwrap_sized(ctx, packets):
    """The host unwrap with every capacity = the header's size (rejected headers: capacity 0)."""
    return _host_unwrap(ctx, packets, [max(s, 0) for s in _sizes(packets)])


def test_gpu_unwrap_packed_fits_exactly_short_and_empty(ctx):
    import torch
    from lz4net_b200 import batch
    inputs = [cases.content(m, n, seed=i).tobytes() for i, m in enumerate(cases.MODELS) for n in (0, 1, 300, 65536)]
    packets = _host_wrap(ctx, inputs, False) + [b"\x01\x02"]                                  # and one malformed packet
    sizes = [len(d) for d in inputs] + [E_FORMAT]
    need = sum(len(d) for d in inputs)
    res, off, h = _unwrap_packed(ctx, packets, need - 1)                                      # one byte short: dst untouched
    assert res == sizes and int(off[-1]) == need and (h == GUARD).all()
    res, off, h = _unwrap_packed(ctx, packets, need)                                          # exactly
    assert res == sizes and b"".join(h[off[i]:off[i + 1]].tobytes() for i in range(len(inputs))) == b"".join(inputs)
    assert (h[need:] == GUARD).all()
    z = torch.full((1,), -7, dtype=torch.int64, device="cuda")                                # n = 0
    e = torch.empty(0, dtype=torch.int64, device="cuda")
    batch.unwrap_packed(ctx, torch.zeros(16, dtype=torch.uint8, device="cuda"), e, e.int(), torch.zeros(16, dtype=torch.uint8, device="cuda"),
                        z, torch.empty(0, dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    assert int(z[0]) == 0


@pytest.mark.parametrize("call", ["wrap", "wrap_hc", "unwrap", "unwrap_packed"])
def test_gpu_calls_are_asynchronous_on_a_non_default_stream(ctx, call):
    """Issued on a non-default stream behind a long kernel: the call returns before its results exist, and the first host
    read after stream.synchronize() sees them."""
    import time
    import torch
    from lz4net_b200 import batch
    inputs = [cases.content("ETEXT", 65536, seed=i).tobytes() for i in range(64)]
    packets = _host_wrap(ctx, inputs, call == "wrap_hc")
    if call.startswith("wrap"):
        buf, so, sl = _src(inputs)
        caps = sl + 8
        do, total = _layout(caps, 0, 0)
        args = [_dev(buf), _dev(so), _dev(sl), torch.empty(total + 16, dtype=torch.uint8, device="cuda"), _dev(do), _dev(caps)]
        want = [len(p) for p in packets]
    else:
        buf, so, sl = _src(packets)
        do, total = _layout([65536] * 64, 0, 0)
        args = [_dev(buf), _dev(so), _dev(sl), torch.empty(total + 16, dtype=torch.uint8, device="cuda")]
        want = [65536] * 64
    out = torch.full((64,), -9, dtype=torch.int32, device="cuda")
    out_off = torch.full((65,), -1, dtype=torch.int64, device="cuda")
    if call == "wrap_hc":                                                                      # (the HC arena is grown here, not under the timer)
        batch.wrap(ctx, *args, out, hc=True)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a = torch.randn(4096, 4096, device="cuda")
        for _ in range(40):
            a = a @ a
            a = a / a.norm()
        t0 = time.perf_counter()
        if call.startswith("wrap"):
            batch.wrap(ctx, *args, out, hc=call == "wrap_hc")
        elif call == "unwrap":
            batch.unwrap(ctx, *args, _dev(do), _dev(np.full(64, 65536, np.int32)), out)
        else:
            batch.unwrap_packed(ctx, *args, out_off, out)
        enqueue = time.perf_counter() - t0
        ev = torch.cuda.Event(); ev.record(s)
    assert not ev.query(), "the call waited for the stream"
    s.synchronize()
    assert out.cpu().tolist() == want
    if call == "unwrap_packed":
        assert int(out_off[64]) == 64 * 65536
    assert enqueue < 0.5


def test_gpu_large_e50_batch_round_trip(ctx):
    """2^17 x 64 KiB E50 blocks: wrapped, packed back to back, unwrapped (slots and packed); the bytes hash equal to the input."""
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 1 << 17, 65536
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID["E50"], seed=33)
    h_raw = hashlib.sha256(raw.cpu().numpy().tobytes()).hexdigest()
    so, do, sl, dc = batch.uniform_layout(nb, bs, bs + 8, "cuda")
    slots = torch.empty(nb * (bs + 8), dtype=torch.uint8, device="cuda")
    plen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    packed = torch.empty(nb * (bs + 8), dtype=torch.uint8, device="cuda")
    poff = torch.zeros(nb + 1, dtype=torch.int64, device="cuda")
    batch.wrap_packed(ctx, raw, so, sl, slots, do, dc, plen, packed, poff)
    torch.cuda.synchronize()
    assert bool((plen > 8).all()) and bool((plen < bs + 8).all())
    del slots
    raw.fill_(0)
    res = torch.zeros(nb, dtype=torch.int32, device="cuda")
    pstart = poff[:-1].contiguous()
    batch.unwrap(ctx, packed, pstart, plen, raw, so, sl, res)
    torch.cuda.synchronize()
    assert bool((res == bs).all())
    assert hashlib.sha256(raw.cpu().numpy().tobytes()).hexdigest() == h_raw
    raw.fill_(0)
    out_off = torch.zeros(nb + 1, dtype=torch.int64, device="cuda")
    batch.unwrap_packed(ctx, packed, pstart, plen, raw, out_off, res)
    torch.cuda.synchronize()
    assert bool((res == bs).all()) and int(out_off[nb]) == nb * bs
    assert hashlib.sha256(raw.cpu().numpy().tobytes()).hexdigest() == h_raw
