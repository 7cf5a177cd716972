"""Wrap / Unwrap packets between device and host memory on an H100: lz4b200_wrap_batch_from_device and its packed form
(inputs in HBM, packets to host memory), lz4b200_unwrap_batch_to_device and its packed form (packets in host memory,
restored into HBM).

Packets must be byte for byte those of the host lz4b200_wrap_batch and of LZ4Codec.Wrap's rule; statuses must be those of
the host lz4b200_unwrap_batch; nothing may be written outside a packet's bytes (host) or an output slot (device); the
calls are ordered behind the work already queued on the caller's stream and refuse the wrong kind of memory."""
import functools
import hashlib
import struct

import numpy as np
import pytest

from tests import cases
from tests.test_mixed_memory_gpu import _busy, _host, _Options, CHUNK_MB_DEFAULT
from tests.test_wrap_device_gpu import _corrupt, _device_unwrap, _host_unwrap, _host_unwrap_sized, _host_wrap, _sizes, _src, ref_wrap

pytestmark = pytest.mark.gpu

LENS = (0, 1, 12, 13, 65535, 65536, 65537, 65547, 1 << 20)
HOST_GUARD, DEV_GUARD = 0xEE, 0xA5
E_ARG, E_FORMAT = -1, -5


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@functools.lru_cache(maxsize=None)
def _ref(d, hc):
    return ref_wrap(d, hc)


def _inputs(skip_mib=False):
    return [cases.content(m, n, seed=50 + i).tobytes() for i, m in enumerate(cases.MODELS) for n in LENS
            if not (skip_mib and n == 1 << 20)]


def _shuffled(sizes, skew, gap, seed=3):
    """int64 offsets of `sizes` laid out in a shuffled order with `gap` bytes between them, the first `skew` bytes in."""
    order = np.random.default_rng(seed).permutation(len(sizes))
    off = np.zeros(len(sizes), np.int64)
    pos = skew
    for i in order:
        off[i] = pos
        pos += max(int(sizes[i]), 0) + gap
    return off, pos


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _wrap_slots(ctx, inputs, hc, pinned):
    """wrap_to_host into host slots with 0-2 spare bytes each, shuffled, misaligned, guard bytes around and between them.
    Returns (out_len, packets); asserts that no byte outside a packet changed."""
    from lz4net_b200 import batch
    buf, so, sl = _src(inputs)
    caps = (sl + 8 + np.arange(len(inputs)) % 3).astype(np.int32)
    do, total = _shuffled(caps, 7, 9)
    dst = _host(total + 64, HOST_GUARD, pinned)
    out = np.full(len(inputs), 12345, np.int32)
    batch.wrap_to_host(ctx, _dev(buf), so, sl, dst, do, caps, out, hc=hc)
    written = np.zeros(len(dst), bool)
    for o, r in zip(do, out):
        written[o:o + max(int(r), 0)] = True
    assert (dst[~written] == HOST_GUARD).all(), "a host byte outside [dst_off, dst_off + out_len) changed"
    return out.tolist(), [dst[o:o + max(int(r), 0)].tobytes() for o, r in zip(do, out)]


def _wrap_packed(ctx, inputs, hc, pinned, room=None):
    """wrap_to_host_packed into a host buffer of `room` bytes (default: sum(len + 8)) with guard bytes behind it."""
    from lz4net_b200 import batch
    buf, so, sl = _src(inputs)
    room = int((sl.astype(np.int64) + 8).sum()) if room is None else room
    dst = _host(room + 64, HOST_GUARD, pinned)
    off = np.full(len(inputs) + 1, -7, np.int64)
    out = np.full(len(inputs), 12345, np.int32)
    total = batch.wrap_to_host_packed(ctx, _dev(buf), so, sl, dst[:room], off, out, hc=hc)
    assert (dst[total:] == HOST_GUARD).all(), "a host byte behind the packed total changed"
    return out.tolist(), off.tolist(), dst[:total].tobytes()


@pytest.mark.parametrize("pinned,chunk_mb", [(False, CHUNK_MB_DEFAULT), (True, 1), (True, CHUNK_MB_DEFAULT)],
                         ids=["pageable-default-stages", "pinned-many-stages", "pinned-default-stages"])
@pytest.mark.parametrize("mode", ["fast", "hc-auto", "hc0", "hc1", "hc2"])
def test_gpu_wrap_to_host_equals_host_and_reference(ctx, mode, pinned, chunk_mb):
    """Every content model at lengths 0 .. 1 MiB from a misaligned device source: into shuffled host slots (n > 8: compacted
    and scattered), into the slots of the first eight (one copy per packet) and packed (appended).  (The thread-per-block
    HC kernel, hc0, skips the 1 MiB inputs: one thread encoding a MiB takes seconds.)"""
    hc = mode != "fast"
    inputs = _inputs(skip_mib=mode == "hc0")
    opts = {"host_chunk_mb": chunk_mb}
    if mode in ("hc0", "hc1", "hc2"):
        opts["hc_kernel"] = int(mode[2])
    with _Options(ctx, **opts):
        want = _host_wrap(ctx, inputs, hc)
        res, pk = _wrap_slots(ctx, inputs, hc, pinned)
        res8, pk8 = _wrap_slots(ctx, inputs[:8], hc, pinned)
        pres, poff, packed = _wrap_packed(ctx, inputs, hc, pinned)
    assert res == [len(p) for p in want] and pk == want, mode
    assert res8 == res[:8] and pk8 == want[:8], mode
    assert pres == res and poff == list(np.concatenate([[0], np.cumsum(res)])) and packed == b"".join(want), mode
    for i, d in enumerate(inputs):
        if not hc or len(d) <= 65547 or chunk_mb == 1:                                     # (the oracle's HC on 1 MiB is slow)
            assert pk[i] == _ref(d, hc), (mode, i, len(d))
    assert sum(len(p) < len(d) + 8 for p, d in zip(pk, inputs)) > 10 and sum(len(p) == len(d) + 8 for p, d in zip(pk, inputs)) > 10


def _unwrap_slots(ctx, packets, caps, pinned=False):
    """unwrap_to_device into shuffled, misaligned device slots with guard bytes around them.  Returns (out_len, outputs)
    and asserts that no device byte outside [dst_off, dst_off + dst_cap) changed."""
    import torch
    from lz4net_b200 import batch
    buf, so, sl = _src(packets, skew=5, gap=3)
    src = _host(len(buf), 0, pinned)
    src[:] = buf
    caps = np.asarray(caps, np.int32)
    do, total = _shuffled(caps, 11, 13, seed=4)
    dst = torch.full((total + 64,), DEV_GUARD, dtype=torch.uint8, device="cuda")
    out = np.full(len(packets), 12345, np.int32)
    batch.unwrap_to_device(ctx, src, so, sl, dst, do, caps, out)
    h = dst.cpu().numpy()
    slot = np.zeros(len(h), bool)
    for o, c in zip(do, caps):
        slot[o:o + max(int(c), 0)] = True
    assert (h[~slot] == DEV_GUARD).all(), "a device byte outside [dst_off, dst_off + dst_cap) changed"
    return out.tolist(), [h[o:o + max(int(r), 0)].tobytes() for o, r in zip(do, out)]


def _unwrap_packed(ctx, packets, room, pinned=False):
    """unwrap_to_device_packed into a device buffer of `room` bytes with guard bytes behind it: (out_len, out_off, bytes)."""
    import torch
    from lz4net_b200 import batch
    buf, so, sl = _src(packets, skew=1, gap=2)
    src = _host(len(buf), 0, pinned)
    src[:] = buf
    n = len(packets)
    dst = torch.full((max(room, 0) + 64,), DEV_GUARD, dtype=torch.uint8, device="cuda")
    off = np.full(n + 1, -7, np.int64)
    out = np.full(n, 12345, np.int32)
    assert batch.unwrap_to_device_packed(ctx, src, so, sl, dst[:room], off, out) == off[n]
    return out.tolist(), off, dst.cpu().numpy()


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("chunk_mb", [1, CHUNK_MB_DEFAULT], ids=["many-stages", "default-stages"])
@pytest.mark.parametrize("hc", [False, True])
def test_gpu_unwrap_to_device_round_trips(ctx, hc, chunk_mb, pinned):
    inputs = _inputs()
    packets = _host_wrap(ctx, inputs, hc)
    with _Options(ctx, host_chunk_mb=chunk_mb):
        res, outs = _unwrap_slots(ctx, packets, [len(d) + i % 3 for i, d in enumerate(inputs)], pinned)
        assert res == [len(d) for d in inputs] and outs == inputs
        res, outs = _unwrap_slots(ctx, packets[:8], [len(d) for d in inputs[:8]], pinned)
        assert res == [len(d) for d in inputs[:8]] and outs == inputs[:8]
        need = sum(len(d) for d in inputs)
        res, off, h = _unwrap_packed(ctx, packets, need, pinned)
    assert res == [len(d) for d in inputs] and off[0] == 0 and int(off[-1]) == need
    assert all(h[off[i]:off[i + 1]].tobytes() == d for i, d in enumerate(inputs))
    assert (h[need:] == DEV_GUARD).all()


def _status_cases(ctx):
    """The rejections of the device-memory tests, plus a compressed payload one byte short (its header says so too)."""
    pairs = _corrupt(ctx)
    for d in (cases.content("ETEXT", 5000, seed=9).tobytes(), cases.content("mixed", 65536, seed=9).tobytes()):
        p = _host_wrap(ctx, [d], False)[0]
        raw, stored = struct.unpack("<ii", p[:8])
        assert stored < raw
        pairs.append((struct.pack("<ii", raw, stored - 1) + p[8:-1], raw))
    pairs.append((struct.pack("<iI", 10, 2 ** 31) + bytes(10), 10))                           # storedLen of 2^31
    pairs.append((struct.pack("<Ii", 2 ** 31 + 5, 3) + bytes(3), 100))                        # rawLen above 2^31
    return pairs


@pytest.mark.parametrize("chunk_mb", [1, CHUNK_MB_DEFAULT], ids=["many-stages", "default-stages"])
def test_gpu_unwrap_to_device_statuses_equal_host(ctx, chunk_mb):
    """Packets of 0-7 bytes, storedLen > n - 8, lengths of 2^31 or more, size-0 packets, payloads cut short, trailing
    bytes, bit flips, a capacity one byte short: statuses and restored bytes equal lz4b200_unwrap_batch's, and both equal
    those of lz4b200_unwrap_batch_device, which reads the headers on the device instead of the host."""
    pairs = _status_cases(ctx)
    packets, caps = [p for p, _ in pairs], [c for _, c in pairs]
    want, wout = _host_unwrap(ctx, packets, caps)
    dev, dout = _device_unwrap(ctx, packets, caps)
    assert dev == want
    for i, w in enumerate(want):
        if w >= 0:
            assert dout[i] == wout[i], i
    with _Options(ctx, host_chunk_mb=chunk_mb):
        got, gout = _unwrap_slots(ctx, packets, caps)
        want_nolimit, wout_nl = _host_unwrap_sized(ctx, packets)
        sizes = [max(s, 0) for s in _sizes(packets)]
        res, off, h = _unwrap_packed(ctx, packets, sum(sizes))
    assert got == want
    for i, w in enumerate(want):
        if w >= 0:
            assert gout[i] == wout[i], i
    assert {E_ARG, E_FORMAT} <= set(want) and sum(w >= 0 for w in want) > 20 and 0 in want
    assert res == want_nolimit and list(np.diff(off)) == sizes
    for i, w in enumerate(want_nolimit):
        if w >= 0:
            assert h[off[i]:off[i] + w].tobytes() == wout_nl[i], i


def test_gpu_unwrap_packed_to_device_fits_exactly_short_and_empty(ctx):
    from lz4net_b200 import batch
    import torch
    inputs = [cases.content(m, n, seed=i).tobytes() for i, m in enumerate(cases.MODELS) for n in (0, 1, 300, 65536)]
    packets = _host_wrap(ctx, inputs, False) + [b"\x01\x02"]                                  # and one malformed packet
    sizes = [len(d) for d in inputs] + [E_FORMAT]
    need = sum(len(d) for d in inputs)
    res, off, h = _unwrap_packed(ctx, packets, need - 1)                                      # one byte short: dst untouched
    assert res == sizes and int(off[-1]) == need and list(np.diff(off)) == [max(s, 0) for s in sizes]
    assert (h == DEV_GUARD).all()
    res, off, h = _unwrap_packed(ctx, packets, need)                                          # exactly
    assert res == sizes and b"".join(h[off[i]:off[i + 1]].tobytes() for i in range(len(inputs))) == b"".join(inputs)
    assert (h[need:] == DEV_GUARD).all()
    z = np.full(1, -7, np.int64)                                                              # n = 0
    e64, e32 = np.zeros(0, np.int64), np.zeros(0, np.int32)
    assert batch.unwrap_to_device_packed(ctx, np.zeros(16, np.uint8), e64, e32, torch.zeros(16, dtype=torch.uint8, device="cuda"),
                                         z, e32) == 0 and z[0] == 0


def test_gpu_wrap_mixed_calls_refuse_bad_arguments_and_the_wrong_kind_of_memory(ctx):
    """E_ARG for a wrap capacity below len + 8 (nothing written), a negative length, a packed destination one byte short,
    the wrong kind of memory on either side of every call; n = 0 is OK."""
    import torch
    from lz4net_b200 import native
    l = native.lib()
    inputs = [cases.content("E50", 1000 + i, seed=i).tobytes() for i in range(4)]
    buf, so, sl = _src(inputs)
    caps = (sl + 8).astype(np.int32)
    do = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
    total = int(caps.sum())
    d_src, h_src = _dev(buf), buf.copy()
    h_dst, d_dst = np.full(total + 16, HOST_GUARD, np.uint8), torch.zeros(total + 16, dtype=torch.uint8, device="cuda")
    out = np.full(4, 12345, np.int32)
    off = np.zeros(5, np.int64)
    p = lambda a: a.ctypes.data                                                              # noqa: E731
    wrap = lambda src, dst, sl_, caps_: l.lz4b200_wrap_batch_from_device(                    # noqa: E731
        ctx.handle, src, p(so), p(sl_), 0, dst, p(do), p(caps_), p(out), 4, 0)
    packed = lambda src, dst, room: l.lz4b200_wrap_batch_packed_from_device(                 # noqa: E731
        ctx.handle, src, p(so), p(sl), 0, dst, room, p(off), p(out), 4, 0)
    short = caps.copy(); short[2] -= 1
    neg = sl.copy(); neg[1] = -1
    assert wrap(d_src.data_ptr(), p(h_dst), sl, short) == E_ARG
    assert wrap(d_src.data_ptr(), p(h_dst), neg, caps) == E_ARG
    assert (h_dst == HOST_GUARD).all() and (out == 12345).all(), "a refused call wrote something"
    assert wrap(p(h_src), p(h_dst), sl, caps) == E_ARG                                       # host src as the device side
    assert wrap(d_src.data_ptr(), d_dst.data_ptr(), sl, caps) == E_ARG                       # device dst as the host side
    assert packed(p(h_src), p(h_dst), total) == E_ARG
    assert packed(d_src.data_ptr(), d_dst.data_ptr(), total) == E_ARG
    assert wrap(d_src.data_ptr(), p(h_dst), sl, caps) == 0                                   # the right sides
    psize = out.copy()
    pk = h_dst.copy()
    assert packed(d_src.data_ptr(), p(h_dst), int(psize.sum())) == 0 and off[4] == psize.sum()
    assert packed(d_src.data_ptr(), p(h_dst), int(psize.sum()) - 1) == E_ARG                 # one byte short
    # unwrap: the packets just made, in host memory
    un = lambda src, dst: l.lz4b200_unwrap_batch_to_device(                                  # noqa: E731
        ctx.handle, src, p(do), p(psize), dst, p(so), p(sl), p(out), 4, 0)
    unp = lambda src, dst: l.lz4b200_unwrap_batch_packed_to_device(                          # noqa: E731
        ctx.handle, src, p(do), p(psize), dst, total, p(off), p(out), 4, 0)
    d_pk = _dev(pk)
    assert un(d_pk.data_ptr(), d_dst.data_ptr()) == E_ARG                                    # device src as the host side
    assert un(p(pk), p(h_dst)) == E_ARG                                                      # host dst as the device side
    assert unp(d_pk.data_ptr(), d_dst.data_ptr()) == E_ARG
    assert unp(p(pk), p(h_dst)) == E_ARG
    assert un(p(pk), d_dst.data_ptr()) == 0 and out.tolist() == sl.tolist()
    assert all(d_dst[int(o):int(o) + int(k)].cpu().numpy().tobytes() == d for o, k, d in zip(so, sl, inputs))
    z = np.full(1, -7, np.int64)
    assert l.lz4b200_wrap_batch_from_device(ctx.handle, None, None, None, 0, None, None, None, None, 0, 0) == 0
    assert l.lz4b200_wrap_batch_packed_from_device(ctx.handle, None, None, None, 0, None, 0, p(z), None, 0, 0) == 0 and z[0] == 0
    assert l.lz4b200_unwrap_batch_to_device(ctx.handle, None, None, None, None, None, None, None, 0, 0) == 0
    z[0] = -7
    assert l.lz4b200_unwrap_batch_packed_to_device(ctx.handle, None, None, None, None, 0, p(z), None, 0, 0) == 0 and z[0] == 0


@pytest.mark.parametrize("hc", [False, True])
def test_gpu_wrap_mixed_packets_interchange_with_host_and_device_calls(ctx, hc):
    """Packets of wrap_batch_device and of the host wrap_batch unwrap through the new calls; the new calls' packets unwrap
    through the host unwrap_batch and unwrap_batch_device."""
    import torch
    from lz4net_b200 import batch
    inputs = _inputs(skip_mib=True)
    buf, so, sl = _src(inputs)
    caps = (sl + 8).astype(np.int32)
    do = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
    slots = torch.zeros(int(caps.sum()) + 16, dtype=torch.uint8, device="cuda")
    plen = torch.zeros(len(inputs), dtype=torch.int32, device="cuda")
    batch.wrap(ctx, _dev(buf), _dev(so), _dev(sl), slots, _dev(do), _dev(caps), plen, hc=hc)
    torch.cuda.synchronize()
    h = slots.cpu().numpy()
    dev_pk = [h[o:o + r].tobytes() for o, r in zip(do, plen.cpu().tolist())]
    host_pk = _host_wrap(ctx, inputs, hc)
    sizes = [len(d) for d in inputs]
    for pk in (dev_pk, host_pk):
        assert _unwrap_slots(ctx, pk, sizes) == (sizes, inputs)
    _, new_pk = _wrap_slots(ctx, inputs, hc, False)
    assert _host_unwrap(ctx, new_pk, sizes) == (sizes, inputs)
    pbuf, pso, psl = _src(new_pk)
    out_t = torch.zeros(sum(sizes) + 16, dtype=torch.uint8, device="cuda")
    oo = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    res = torch.zeros(len(inputs), dtype=torch.int32, device="cuda")
    batch.unwrap(ctx, _dev(pbuf), _dev(pso), _dev(psl), out_t, _dev(oo), _dev(np.array(sizes, np.int32)), res)
    torch.cuda.synchronize()
    assert res.cpu().tolist() == sizes and out_t[:sum(sizes)].cpu().numpy().tobytes() == b"".join(inputs)


def test_gpu_wrap_to_host_waits_for_the_producer_on_its_stream(ctx):
    """synth_fill queued on a non-default stream behind a long kernel chain, then at once a packed wrap given that stream:
    the packets are those of the filled data, the same as after a synchronise."""
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 256, 65536
    so = np.arange(nb, dtype=np.int64) * bs
    sl = np.full(nb, bs, np.int32)

    def run(sync):
        raw = torch.zeros(nb * bs, dtype=torch.uint8, device="cuda")
        dst = np.zeros(nb * (bs + 8), np.uint8)
        off, out = np.zeros(nb + 1, np.int64), np.zeros(nb, np.int32)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        _busy(s)
        with torch.cuda.stream(s):
            batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID["E50"], seed=7)
            if sync:
                s.synchronize()
            w = batch.wrap_to_host_packed(ctx, raw, so, sl, dst, off, out)
        return dst[:w].tobytes(), raw

    p0, _ = run(False)
    p1, raw = run(True)
    assert p0 == p1 and len(p1) < nb * bs * 0.9                                               # E50 data, not zeros
    host = raw.cpu().numpy()
    assert p1[:200] == _host_wrap(ctx, [host[:bs].tobytes()], False)[0][:200]


def test_gpu_unwrap_to_device_waits_for_readers_of_the_old_contents(ctx):
    """A dst.clone() queued on a non-default stream behind a long kernel chain, then at once an unwrap into dst given that
    stream: the clone holds the old contents, not the restored bytes."""
    import torch
    from lz4net_b200 import batch
    inputs = [cases.content("ETEXT", 65536, seed=i).tobytes() for i in range(64)]
    packets = _host_wrap(ctx, inputs, False)
    buf, so, sl = _src(packets)
    do = np.arange(64, dtype=np.int64) * 65536
    caps = np.full(64, 65536, np.int32)
    dst = torch.full((64 * 65536,), 0x5A, dtype=torch.uint8, device="cuda")
    res = np.zeros(64, np.int32)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    _busy(s)
    with torch.cuda.stream(s):
        snap = dst.clone()
        batch.unwrap_to_device(ctx, buf, so, sl, dst, do, caps, res)
    s.synchronize()
    assert bool((snap == 0x5A).all()), "the unwrap overwrote dst before an earlier reader on the stream was done"
    assert res.tolist() == [65536] * 64 and dst.cpu().numpy().tobytes() == b"".join(inputs)


def test_gpu_large_e50_round_trip_through_host_packets(ctx):
    """2^17 x 64 KiB E50 inputs: packed wrap into host memory, packed unwrap back into HBM; the bytes hash equal."""
    import torch
    from lz4net_b200 import batch, synth
    nb, bs = 1 << 17, 65536
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID["E50"], seed=33)
    h_raw = hashlib.sha256(raw.cpu().numpy().tobytes()).hexdigest()
    so = np.arange(nb, dtype=np.int64) * bs
    sl = np.full(nb, bs, np.int32)
    wire = np.empty(nb * (bs + 8), np.uint8)
    off, plen = np.zeros(nb + 1, np.int64), np.zeros(nb, np.int32)
    total = batch.wrap_to_host_packed(ctx, raw, so, sl, wire, off, plen)
    assert (plen > 8).all() and (plen < bs + 8).all() and total == int(plen.astype(np.int64).sum())
    raw.fill_(0)
    out_off, res = np.zeros(nb + 1, np.int64), np.zeros(nb, np.int32)
    assert batch.unwrap_to_device_packed(ctx, wire, off[:-1].copy(), plen, raw, out_off, res) == nb * bs
    assert (res == bs).all() and np.array_equal(out_off, np.arange(nb + 1, dtype=np.int64) * bs)
    assert hashlib.sha256(raw.cpu().numpy().tobytes()).hexdigest() == h_raw


def test_gpu_wrap_mixed_device_memory_is_flat_in_the_batch_size(ctx):
    """The device memory a fresh context adds for a packed wrap and a packed unwrap of 256 MiB and of 1 GiB of E50 differs
    by less than one pipeline stage, and stays below half the batch.  (32 MiB stages: both batches keep all three pipeline
    slots full, so the scratch has reached its size in both.)"""
    import torch
    import lz4net_b200
    from lz4net_b200 import batch, synth
    bs, stage_mb = 65536, 32
    added = {}
    for mib in (256, 1024):
        nb = (mib << 20) // bs
        raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
        batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID["E50"], seed=mib)
        so = np.arange(nb, dtype=np.int64) * bs
        sl = np.full(nb, bs, np.int32)
        wire = torch.empty(nb * (bs + 8), dtype=torch.uint8).pin_memory().numpy()
        off, plen, res = np.zeros(nb + 1, np.int64), np.zeros(nb, np.int32), np.zeros(nb, np.int32)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        c = lz4net_b200.Context(0)
        c.set_option("host_chunk_mb", stage_mb)
        batch.wrap_to_host_packed(c, raw, so, sl, wire, off, plen)
        batch.unwrap_to_device_packed(c, wire, off[:-1].copy(), plen, raw, np.zeros(nb + 1, np.int64), res)
        torch.cuda.synchronize()
        added[mib] = free0 - torch.cuda.mem_get_info()[0]
        c.close()
        assert (res == bs).all()
        del raw
        torch.cuda.empty_cache()
    assert abs(added[1024] - added[256]) < stage_mb << 20, added
    assert added[1024] < 512 << 20, added


@pytest.mark.parametrize("hc", [False, True])
def test_gpu_lz4codec_wrap_of_a_cuda_tensor_equals_wrap_of_its_bytes(ctx, hc):
    import torch
    from lz4net_b200 import LZ4Codec
    wrap = LZ4Codec.WrapHC if hc else LZ4Codec.Wrap
    for m, n in (("ETEXT", 100000), ("E100", 5000), ("runs", 13), ("E50", 0), ("mixed", 65547)):
        d = cases.content(m, n, seed=12).tobytes()
        t = _dev(np.frombuffer(d, np.uint8).copy())
        assert wrap(t) == wrap(d), (m, n)
        if n > 7:
            assert wrap(t, 7, 300) == wrap(d, 7, 300), (m, n)
        assert LZ4Codec.Unwrap(wrap(t)) == d
    f = torch.arange(1000, dtype=torch.float32, device="cuda")                                 # any dtype: its bytes
    assert wrap(f) == wrap(f.cpu().numpy().tobytes())
