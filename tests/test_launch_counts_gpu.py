"""The kernel launches each call family enqueues, on an H100, and the context's shared call scratch across streams.

The launch counts (`lz4b200_launch_count` before and after a call) pin what every call runs on a small fixed input: the
encoders, decoders and measure pass in every kind of memory a call accepts, host batches of one block and of more than
eight (every landing mode of the host pipeline), every pinned `decode_lanes` value and the automatic pick, the LZ4Stream
and Wrap / Unwrap calls in their host, device, mixed and packed forms, and the packed decode into device memory over
several pipeline stages; and the six asynchronous calls between device memory and page-locked host memory in one stage and
in several.  A change to the host code that adds, drops or reorders a step shows up here.

The device calls share the context's scan scratch, capacities and packet view whatever stream they are on.  Enqueued on
two streams with no synchronise in between, a call that grows that scratch and one that does not must both give their
results."""
import numpy as np
import pytest

import oracle
from tests import cases
from tests.test_mixed_memory_gpu import _dev, _layout, _src

pytestmark = pytest.mark.gpu

LANES = (1, 4, 8, 16, 32, 104, 108, 116, 132)
MEMS = {"host": 0, "device": 1, "device_to_host": 2, "host_to_device": 3}

# Recorded on an H100 80GB HBM3; the same before and after the host pipeline named its operations and stage kinds, and
# (the asynchronous rows) before and after the pipeline's stage kinds were dispatched in one place.
EXPECTED = {
    'encode/fast/host/1': 1, 'encode/hc/host/1': 2, 'decode/known/host/1': 1, 'decode/unknown/host/1': 1,
    'encode/fast/device/1': 1, 'encode/hc/device/1': 3, 'decode/known/device/1': 5, 'decode/unknown/device/1': 5,
    'encode/fast/device_to_host/1': 1, 'encode/hc/device_to_host/1': 2, 'decode/known/device_to_host/1': 1,
    'decode/unknown/device_to_host/1': 1, 'encode/fast/host_to_device/1': 1, 'encode/hc/host_to_device/1': 2,
    'decode/known/host_to_device/1': 1, 'decode/unknown/host_to_device/1': 1, 'measure/known/host/1': 1,
    'measure/unknown/host/1': 1, 'measure/known/device/1': 1, 'measure/unknown/device/1': 1,
    'encode_packed/fast/host/1': 5, 'encode_packed/fast/device_to_host/1': 5, 'encode_packed/hc/host/1': 6,
    'encode_packed/hc/device_to_host/1': 6, 'stream_encode/fast/host/1': 6, 'stream_encode/fast/device_to_host/1': 6,
    'stream_encode/hc/host/1': 7, 'stream_encode/hc/device_to_host/1': 7, 'stream_decode/fast/host/1': 2,
    'stream_decode/fast/host_to_device/1': 2, 'stream_decode/hc/host/1': 2, 'stream_decode/hc/host_to_device/1': 2,
    'wrap/fast/host/1': 3, 'wrap/fast/device_to_host/1': 3, 'wrap_packed/fast/device_to_host/1': 7,
    'wrap/fast/device/1': 3, 'wrap/hc/host/1': 4, 'wrap/hc/device_to_host/1': 4, 'wrap_packed/hc/device_to_host/1': 8,
    'wrap/hc/device/1': 5, 'unwrap/fast/host/1': 2, 'unwrap/fast/host_to_device/1': 2,
    'unwrap_packed/fast/host_to_device/1': 2, 'unwrap/fast/device/1': 7, 'unwrap_packed/fast/device/1': 11,
    'unwrap/hc/host/1': 2, 'unwrap/hc/host_to_device/1': 2, 'unwrap_packed/hc/host_to_device/1': 2,
    'unwrap/hc/device/1': 7, 'unwrap_packed/hc/device/1': 11, 'encode/fast/host/12': 5, 'encode/hc/host/12': 6,
    'decode/known/host/12': 1, 'decode/unknown/host/12': 5, 'encode/fast/device/12': 1, 'encode/hc/device/12': 3,
    'decode/known/device/12': 5, 'decode/unknown/device/12': 5, 'encode/fast/device_to_host/12': 5,
    'encode/hc/device_to_host/12': 6, 'decode/known/device_to_host/12': 1, 'decode/unknown/device_to_host/12': 5,
    'encode/fast/host_to_device/12': 1, 'encode/hc/host_to_device/12': 2, 'decode/known/host_to_device/12': 1,
    'decode/unknown/host_to_device/12': 1, 'measure/known/host/12': 1, 'measure/unknown/host/12': 1,
    'measure/known/device/12': 1, 'measure/unknown/device/12': 1, 'encode_packed/fast/host/12': 5,
    'encode_packed/fast/device_to_host/12': 5, 'encode_packed/hc/host/12': 6, 'encode_packed/hc/device_to_host/12': 6,
    'stream_encode/fast/host/12': 6, 'stream_encode/fast/device_to_host/12': 6, 'stream_encode/hc/host/12': 7,
    'stream_encode/hc/device_to_host/12': 7, 'stream_decode/fast/host/12': 2, 'stream_decode/fast/host_to_device/12': 2,
    'stream_decode/hc/host/12': 2, 'stream_decode/hc/host_to_device/12': 2, 'wrap/fast/host/12': 7,
    'wrap/fast/device_to_host/12': 7, 'wrap_packed/fast/device_to_host/12': 7, 'wrap/fast/device/12': 3,
    'wrap/hc/host/12': 8, 'wrap/hc/device_to_host/12': 8, 'wrap_packed/hc/device_to_host/12': 8, 'wrap/hc/device/12': 5,
    'unwrap/fast/host/12': 2, 'unwrap/fast/host_to_device/12': 2, 'unwrap_packed/fast/host_to_device/12': 2,
    'unwrap/fast/device/12': 7, 'unwrap_packed/fast/device/12': 11, 'unwrap/hc/host/12': 2,
    'unwrap/hc/host_to_device/12': 2, 'unwrap_packed/hc/host_to_device/12': 2, 'unwrap/hc/device/12': 7,
    'unwrap_packed/hc/device/12': 11, 'decode/known/device/auto': 5, 'decode/unknown/device/auto': 5,
    'decode_batch_packed/auto': 10, 'decode/known/device/lanes1': 1, 'decode/unknown/device/lanes1': 1,
    'decode_batch_packed/lanes1': 7, 'decode/known/device/lanes4': 1, 'decode/unknown/device/lanes4': 1,
    'decode_batch_packed/lanes4': 7, 'decode/known/device/lanes8': 1, 'decode/unknown/device/lanes8': 1,
    'decode_batch_packed/lanes8': 7, 'decode/known/device/lanes16': 1, 'decode/unknown/device/lanes16': 1,
    'decode_batch_packed/lanes16': 7, 'decode/known/device/lanes32': 1, 'decode/unknown/device/lanes32': 1,
    'decode_batch_packed/lanes32': 7, 'decode/known/device/lanes104': 1, 'decode/unknown/device/lanes104': 1,
    'decode_batch_packed/lanes104': 7, 'decode/known/device/lanes108': 1, 'decode/unknown/device/lanes108': 1,
    'decode_batch_packed/lanes108': 7, 'decode/known/device/lanes116': 1, 'decode/unknown/device/lanes116': 1,
    'decode_batch_packed/lanes116': 7, 'decode/known/device/lanes132': 1, 'decode/unknown/device/lanes132': 1,
    'decode_batch_packed/lanes132': 7, 'decode_packed/host_to_device/auto': 30,
    'decode_packed/host_to_device/lanes16': 21,
    'encode_packed_async/fast/1stage': 5, 'wrap_packed_async/fast/1stage': 7, 'encode_packed_async/hc/1stage': 7,
    'wrap_packed_async/hc/1stage': 9, 'decode_async/known/1stage': 1, 'decode_async/unknown/1stage': 1,
    'decode_packed_async/1stage': 10, 'unwrap_async/fast/1stage': 7, 'unwrap_packed_async/fast/1stage': 11,
    'unwrap_async/hc/1stage': 7, 'unwrap_packed_async/hc/1stage': 11, 'encode_packed_async/fast/stages': 20,
    'wrap_packed_async/fast/stages': 28, 'encode_packed_async/hc/stages': 28, 'wrap_packed_async/hc/stages': 36,
    'decode_async/known/stages': 3, 'decode_async/unknown/stages': 3, 'decode_packed_async/stages': 30,
    'unwrap_async/fast/stages': 21, 'unwrap_packed_async/fast/stages': 33, 'unwrap_async/hc/stages': 14,
    'unwrap_packed_async/hc/stages': 22,
}


@pytest.fixture()
def ctx():
    import lz4net_b200
    c = lz4net_b200.Context(0)                            # a context of its own: library defaults, empty scratch
    yield c
    c.close()


def _raws(n, size=16384):
    """n blocks of size bytes, content models in turn (E0 first: stored by the Wrap and LZ4Stream rules)."""
    return [cases.content(cases.MODELS[i % len(cases.MODELS)], size, seed=300 + i).tobytes() for i in range(n)]


class _Counter:
    def __init__(self, ctx):
        self.ctx, self.counts = ctx, {}

    def __call__(self, name, fn):
        import torch
        torch.cuda.synchronize()
        before = self.ctx.launches
        rc = fn()
        torch.cuda.synchronize()
        assert rc is None or rc >= 0, (name, rc)
        self.counts[name] = self.ctx.launches - before
        return rc


def _ptr(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def _batch_calls(ctx, count, n):
    """encode / decode / measure batches of n blocks in every kind of memory, and the packed encodes."""
    import torch
    from lz4net_b200 import native
    lib, h, st = native.lib(), ctx.handle, torch.cuda.current_stream().cuda_stream
    raws = _raws(n)
    comp = [oracle.encode(d)[1] for d in raws]
    rbuf, rso, rsl = _src(raws)
    cbuf, cso, csl = _src(comp)
    ecap = np.array([oracle.bound(len(d)) for d in raws], np.int32)
    edo, etotal = _layout(ecap, 0, 0)
    dcap = np.array([len(d) for d in raws], np.int32)
    ddo, dtotal = _layout(dcap, 0, 0)
    for mem, m in MEMS.items():
        src_dev, dst_dev = m in (1, 2), m in (1, 3)
        for hc in (False, True):
            src = _dev(rbuf) if src_dev else rbuf
            so, sl = (_dev(rso), _dev(rsl)) if m == 1 else (rso, rsl)
            dst = torch.zeros(etotal + 64, dtype=torch.uint8, device="cuda") if dst_dev else np.zeros(etotal + 64, np.uint8)
            do, dc = (_dev(edo), _dev(ecap)) if m == 1 else (edo, ecap)
            out = torch.zeros(n, dtype=torch.int32, device="cuda") if m == 1 else np.zeros(n, np.int32)
            count(f"encode/{'hc' if hc else 'fast'}/{mem}/{n}", lambda: native.check(lib.lz4b200_encode_batch(
                h, _ptr(src), _ptr(so), _ptr(sl), _ptr(dst), _ptr(do), _ptr(dc), _ptr(out), n, int(hc), m, st), "encode"))
        for known in (True, False):
            src = _dev(cbuf) if src_dev else cbuf
            so, sl = (_dev(cso), _dev(csl)) if m == 1 else (cso, csl)
            dst = torch.zeros(dtotal + 64, dtype=torch.uint8, device="cuda") if dst_dev else np.zeros(dtotal + 64, np.uint8)
            do, dc = (_dev(ddo), _dev(dcap)) if m == 1 else (ddo, dcap)
            out = torch.zeros(n, dtype=torch.int32, device="cuda") if m == 1 else np.zeros(n, np.int32)
            count(f"decode/{'known' if known else 'unknown'}/{mem}/{n}", lambda: native.check(lib.lz4b200_decode_batch(
                h, _ptr(src), _ptr(so), _ptr(sl), _ptr(dst), _ptr(do), _ptr(dc), _ptr(out), n, int(known), m, st), "decode"))
            res = out.cpu().numpy() if m == 1 else out
            assert res.tolist() == ([len(c) for c in comp] if known else [len(d) for d in raws]), (mem, known)
    for mem, m in (("host", 0), ("device", 1)):
        for known in (True, False):
            src, so, sl, dc = (_dev(cbuf), _dev(cso), _dev(csl), _dev(dcap)) if m else (cbuf, cso, csl, dcap)
            out = torch.zeros(n, dtype=torch.int32, device="cuda") if m else np.zeros(n, np.int32)
            count(f"measure/{'known' if known else 'unknown'}/{mem}/{n}", lambda: native.check(lib.lz4b200_measure_batch(
                h, _ptr(src), _ptr(so), _ptr(sl), _ptr(dc), _ptr(out), n, int(known), m, st), "measure"))
    for hc in (False, True):
        dst, off, out = np.zeros(etotal + 64, np.uint8), np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
        count(f"encode_packed/{'hc' if hc else 'fast'}/host/{n}", lambda: native.check(lib.lz4b200_encode_batch_packed(
            h, rbuf.ctypes.data, rso.ctypes.data, rsl.ctypes.data, ecap.ctypes.data, dst.ctypes.data, etotal, off.ctypes.data,
            out.ctypes.data, n, int(hc)), "encode_packed"))
        d_raw = _dev(rbuf)
        count(f"encode_packed/{'hc' if hc else 'fast'}/device_to_host/{n}", lambda: native.check(
            lib.lz4b200_encode_batch_packed_from_device(h, d_raw.data_ptr(), rso.ctypes.data, rsl.ctypes.data, ecap.ctypes.data,
                                                        dst.ctypes.data, etotal, off.ctypes.data, out.ctypes.data, n, int(hc), st),
            "encode_packed_from_device"))


def _decoder_calls(ctx, count):
    """A MEM_DEVICE decode and lz4b200_decode_batch_packed with the decoder picked on the device and with every pinned one."""
    import torch
    from lz4net_b200 import native
    lib, h, st = native.lib(), ctx.handle, torch.cuda.current_stream().cuda_stream
    raws = _raws(24)
    comp = [oracle.encode(d)[1] for d in raws]
    buf, so, sl = _src(comp)
    cap = np.array([len(d) for d in raws], np.int32)
    do, total = _layout(cap, 0, 0)
    d_buf, d_so, d_sl, d_do, d_cap = _dev(buf), _dev(so), _dev(sl), _dev(do), _dev(cap)
    for lanes in (0,) + LANES:
        ctx.set_option("decode_lanes", lanes) if lanes else ctx.set_option("decode_lanes_auto", 1)
        name = f"lanes{lanes}" if lanes else "auto"
        for known in (True, False):
            dst = torch.zeros(total, dtype=torch.uint8, device="cuda")
            out = torch.zeros(24, dtype=torch.int32, device="cuda")
            count(f"decode/{'known' if known else 'unknown'}/device/{name}", lambda: native.check(lib.lz4b200_decode_batch(
                h, d_buf.data_ptr(), d_so.data_ptr(), d_sl.data_ptr(), dst.data_ptr(), d_do.data_ptr(), d_cap.data_ptr(),
                out.data_ptr(), 24, int(known), 1, st), "decode"))
            assert dst.cpu().numpy().tobytes() == b"".join(raws), (name, known)
        dst = torch.zeros(total, dtype=torch.uint8, device="cuda")
        off = torch.zeros(25, dtype=torch.int64, device="cuda")
        out = torch.zeros(24, dtype=torch.int32, device="cuda")
        count(f"decode_batch_packed/{name}", lambda: native.check(lib.lz4b200_decode_batch_packed(
            h, d_buf.data_ptr(), d_so.data_ptr(), d_sl.data_ptr(), dst.data_ptr(), total, off.data_ptr(), out.data_ptr(), 24, st),
            "decode_batch_packed"))
        assert dst.cpu().numpy().tobytes() == b"".join(raws), name
    ctx.set_option("decode_lanes_auto", 1)


def _framing_calls(ctx, count, n):
    """LZ4Stream and Wrap / Unwrap calls: host, device, mixed and packed forms."""
    import torch
    from lz4net_b200 import native
    lib, h, st = native.lib(), ctx.handle, torch.cuda.current_stream().cuda_stream
    raws = _raws(n, 12000)
    data = np.frombuffer(b"".join(raws), np.uint8).copy()
    d_data = _dev(data)
    bound = int(lib.lz4b200_stream_bound(len(data), 4096))
    wires = {}
    for hc in (False, True):
        tag = "hc" if hc else "fast"
        wire = np.zeros(bound, np.uint8)
        w = count(f"stream_encode/{tag}/host/{n}",
                  lambda: lib.lz4b200_stream_encode(h, data.ctypes.data, len(data), 4096, int(hc), wire.ctypes.data, bound))
        wire2 = np.zeros(bound, np.uint8)
        count(f"stream_encode/{tag}/device_to_host/{n}", lambda: lib.lz4b200_stream_encode_from_device(
            h, d_data.data_ptr(), len(data), 4096, int(hc), wire2.ctypes.data, bound, st))
        assert wire.tobytes() == wire2.tobytes(), hc
        wires[hc] = wire[:w]
    for hc, wire in wires.items():
        tag = "hc" if hc else "fast"
        back = np.zeros(len(data), np.uint8)
        count(f"stream_decode/{tag}/host/{n}",
              lambda: lib.lz4b200_stream_decode(h, wire.ctypes.data, len(wire), back.ctypes.data, len(back)))
        assert back.tobytes() == data.tobytes()
        d_back = torch.zeros(len(data), dtype=torch.uint8, device="cuda")
        count(f"stream_decode/{tag}/host_to_device/{n}", lambda: lib.lz4b200_stream_decode_to_device(
            h, wire.ctypes.data, len(wire), d_back.data_ptr(), len(data), st))
        assert d_back.cpu().numpy().tobytes() == data.tobytes()

    buf, so, sl = _src(raws)
    d_buf, d_so, d_sl = _dev(buf), _dev(so), _dev(sl)
    caps = sl + 8
    do, total = _layout(caps, 0, 0)
    d_do, d_caps = _dev(do), _dev(caps)
    packets = {}
    for hc in (False, True):
        tag = "hc" if hc else "fast"
        dst, out = np.zeros(total + 64, np.uint8), np.zeros(n, np.int32)
        count(f"wrap/{tag}/host/{n}", lambda: native.check(lib.lz4b200_wrap_batch(
            h, buf.ctypes.data, so.ctypes.data, sl.ctypes.data, int(hc), dst.ctypes.data, do.ctypes.data, caps.ctypes.data,
            out.ctypes.data, n), "wrap_batch"))
        packets[hc] = [dst[o:o + r].tobytes() for o, r in zip(do, out)]
        dst2, out2 = np.zeros(total + 64, np.uint8), np.zeros(n, np.int32)
        count(f"wrap/{tag}/device_to_host/{n}", lambda: native.check(lib.lz4b200_wrap_batch_from_device(
            h, d_buf.data_ptr(), so.ctypes.data, sl.ctypes.data, int(hc), dst2.ctypes.data, do.ctypes.data, caps.ctypes.data,
            out2.ctypes.data, n, st), "wrap_batch_from_device"))
        assert [dst2[o:o + r].tobytes() for o, r in zip(do, out2)] == packets[hc]
        dst3, off3, out3 = np.zeros(total + 64, np.uint8), np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
        count(f"wrap_packed/{tag}/device_to_host/{n}", lambda: native.check(lib.lz4b200_wrap_batch_packed_from_device(
            h, d_buf.data_ptr(), so.ctypes.data, sl.ctypes.data, int(hc), dst3.ctypes.data, total, off3.ctypes.data,
            out3.ctypes.data, n, st), "wrap_batch_packed_from_device"))
        assert dst3[:off3[n]].tobytes() == b"".join(packets[hc])
        d_dst, d_out = torch.zeros(total + 64, dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
        count(f"wrap/{tag}/device/{n}", lambda: native.check(lib.lz4b200_wrap_batch_device(
            h, d_buf.data_ptr(), d_so.data_ptr(), d_sl.data_ptr(), int(hc), d_dst.data_ptr(), d_do.data_ptr(), d_caps.data_ptr(),
            d_out.data_ptr(), n, st), "wrap_batch_device"))
        hd = d_dst.cpu().numpy()
        assert [hd[o:o + r].tobytes() for o, r in zip(do, d_out.cpu().tolist())] == packets[hc]

    for hc, pk in packets.items():
        tag = "hc" if hc else "fast"
        pbuf, pso, psl = _src(pk)
        d_pbuf, d_pso, d_psl = _dev(pbuf), _dev(pso), _dev(psl)
        rcap = np.array([len(d) for d in raws], np.int32)
        rdo, rtotal = _layout(rcap, 0, 0)
        d_rdo, d_rcap = _dev(rdo), _dev(rcap)
        want = b"".join(raws)
        dst, out = np.zeros(rtotal + 64, np.uint8), np.zeros(n, np.int32)
        count(f"unwrap/{tag}/host/{n}", lambda: native.check(lib.lz4b200_unwrap_batch(
            h, pbuf.ctypes.data, pso.ctypes.data, psl.ctypes.data, dst.ctypes.data, rdo.ctypes.data, rcap.ctypes.data,
            out.ctypes.data, n), "unwrap_batch"))
        assert dst[:rtotal].tobytes() == want
        d_dst, out = torch.zeros(rtotal, dtype=torch.uint8, device="cuda"), np.zeros(n, np.int32)
        count(f"unwrap/{tag}/host_to_device/{n}", lambda: native.check(lib.lz4b200_unwrap_batch_to_device(
            h, pbuf.ctypes.data, pso.ctypes.data, psl.ctypes.data, d_dst.data_ptr(), rdo.ctypes.data, rcap.ctypes.data,
            out.ctypes.data, n, st), "unwrap_batch_to_device"))
        assert d_dst.cpu().numpy().tobytes() == want
        d_dst, off, out = torch.zeros(rtotal, dtype=torch.uint8, device="cuda"), np.zeros(n + 1, np.int64), np.zeros(n, np.int32)
        count(f"unwrap_packed/{tag}/host_to_device/{n}", lambda: native.check(lib.lz4b200_unwrap_batch_packed_to_device(
            h, pbuf.ctypes.data, pso.ctypes.data, psl.ctypes.data, d_dst.data_ptr(), rtotal, off.ctypes.data, out.ctypes.data,
            n, st), "unwrap_batch_packed_to_device"))
        assert d_dst.cpu().numpy().tobytes() == want
        d_dst, d_out = torch.zeros(rtotal, dtype=torch.uint8, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
        count(f"unwrap/{tag}/device/{n}", lambda: native.check(lib.lz4b200_unwrap_batch_device(
            h, d_pbuf.data_ptr(), d_pso.data_ptr(), d_psl.data_ptr(), d_dst.data_ptr(), d_rdo.data_ptr(), d_rcap.data_ptr(),
            d_out.data_ptr(), n, st), "unwrap_batch_device"))
        assert d_dst.cpu().numpy().tobytes() == want
        d_dst = torch.zeros(rtotal, dtype=torch.uint8, device="cuda")
        d_off, d_out = torch.zeros(n + 1, dtype=torch.int64, device="cuda"), torch.zeros(n, dtype=torch.int32, device="cuda")
        count(f"unwrap_packed/{tag}/device/{n}", lambda: native.check(lib.lz4b200_unwrap_batch_packed(
            h, d_pbuf.data_ptr(), d_pso.data_ptr(), d_psl.data_ptr(), d_dst.data_ptr(), rtotal, d_off.data_ptr(),
            d_out.data_ptr(), n, st), "unwrap_batch_packed"))
        assert d_dst.cpu().numpy().tobytes() == want


def _placed_calls(ctx, count):
    """lz4b200_decode_batch_packed_to_device over several 1 MiB pipeline stages."""
    import torch
    from lz4net_b200 import native
    lib, h, st = native.lib(), ctx.handle, torch.cuda.current_stream().cuda_stream
    raws = [cases.content(("E0", "E50", "ETEXT")[i % 3], 300000, seed=400 + i).tobytes() for i in range(12)]
    comp = [oracle.encode(d)[1] for d in raws]
    buf, so, sl = _src(comp)
    total = sum(len(d) for d in raws)
    ctx.set_option("host_chunk_mb", 1)
    try:
        for lanes in (0, 16):
            ctx.set_option("decode_lanes", lanes) if lanes else ctx.set_option("decode_lanes_auto", 1)
            dst = torch.zeros(total, dtype=torch.uint8, device="cuda")
            off, out = np.zeros(13, np.int64), np.zeros(12, np.int32)
            count(f"decode_packed/host_to_device/{'lanes16' if lanes else 'auto'}", lambda: native.check(
                lib.lz4b200_decode_batch_packed_to_device(h, buf.ctypes.data, so.ctypes.data, sl.ctypes.data, dst.data_ptr(),
                                                          total, off.ctypes.data, out.ctypes.data, 12, st),
                "decode_batch_packed_to_device"))
            assert dst.cpu().numpy().tobytes() == b"".join(raws) and int(off[12]) == total
    finally:
        ctx.set_option("host_chunk_mb", 128)
        ctx.set_option("decode_lanes_auto", 1)


def _async_calls(ctx, count):
    """The six asynchronous calls between device memory and page-locked host memory, each in one stage (the default
    host_chunk_mb) and over several 1 MiB stages, in fast and HC where the call takes a mode."""
    import torch
    from lz4net_b200 import native
    lib, h, st = native.lib(), ctx.handle, torch.cuda.current_stream().cuda_stream
    raws = [cases.content(("E0", "E50", "ETEXT")[i % 3], 300000, seed=500 + i).tobytes() for i in range(12)]
    n, want = len(raws), b"".join(raws)
    rbuf, rso, rsl = _src(raws)
    d_raw = _dev(rbuf)
    ecap = np.array([oracle.bound(len(d)) for d in raws], np.int32)
    rcap = rsl.copy()
    rdo, rtotal = _layout(rcap, 0, 0)
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()            # noqa: E731
    outs = lambda: (torch.zeros(n + 1, dtype=torch.int64, device="cuda"),             # noqa: E731
                    torch.zeros(n, dtype=torch.int32, device="cuda"))
    cbuf, cso, csl = _src([oracle.encode(d)[1] for d in raws])
    comp = pin(cbuf)
    try:
        for stages, mb in (("1stage", 128), ("stages", 1)):
            ctx.set_option("host_chunk_mb", mb)
            packets = {}
            for hc in (False, True):
                tag = "hc" if hc else "fast"
                dst = pin(np.zeros(int(ecap.sum()) + 64, np.uint8))
                off, out = outs()
                count(f"encode_packed_async/{tag}/{stages}", lambda: native.check(
                    lib.lz4b200_encode_batch_packed_from_device_async(
                        h, d_raw.data_ptr(), rso.ctypes.data, rsl.ctypes.data, ecap.ctypes.data, dst.data_ptr(), dst.numel(),
                        off.data_ptr(), out.data_ptr(), n, int(hc), st), "encode_packed_async"))
                assert int(off[n]) <= dst.numel(), (stages, tag)
                dst = pin(np.zeros(int(rsl.sum()) + 8 * n + 64, np.uint8))
                off, out = outs()
                count(f"wrap_packed_async/{tag}/{stages}", lambda: native.check(lib.lz4b200_wrap_batch_packed_from_device_async(
                    h, d_raw.data_ptr(), rso.ctypes.data, rsl.ctypes.data, int(hc), dst.data_ptr(), dst.numel(), off.data_ptr(),
                    out.data_ptr(), n, st), "wrap_packed_async"))
                packets[hc] = (dst, off.cpu().numpy(), out.cpu().numpy())
            for known in (True, False):
                d_dst, (_, out) = torch.zeros(rtotal, dtype=torch.uint8, device="cuda"), outs()
                count(f"decode_async/{'known' if known else 'unknown'}/{stages}", lambda: native.check(
                    lib.lz4b200_decode_batch_to_device_async(
                        h, comp.data_ptr(), cso.ctypes.data, csl.ctypes.data, d_dst.data_ptr(), rdo.ctypes.data, rcap.ctypes.data,
                        out.data_ptr(), n, int(known), st), "decode_async"))
                assert d_dst.cpu().numpy().tobytes() == want, (stages, known)
            d_dst, (off, out) = torch.zeros(rtotal, dtype=torch.uint8, device="cuda"), outs()
            count(f"decode_packed_async/{stages}", lambda: native.check(lib.lz4b200_decode_batch_packed_to_device_async(
                h, comp.data_ptr(), cso.ctypes.data, csl.ctypes.data, d_dst.data_ptr(), rtotal, off.data_ptr(), out.data_ptr(),
                n, st), "decode_packed_async"))
            assert d_dst.cpu().numpy().tobytes() == want and int(off[n]) == rtotal, stages
            for hc, (pk, poff, plen) in packets.items():
                tag = "hc" if hc else "fast"
                pso = np.ascontiguousarray(poff[:n])
                d_dst, (_, out) = torch.zeros(rtotal, dtype=torch.uint8, device="cuda"), outs()
                count(f"unwrap_async/{tag}/{stages}", lambda: native.check(lib.lz4b200_unwrap_batch_to_device_async(
                    h, pk.data_ptr(), pso.ctypes.data, plen.ctypes.data, d_dst.data_ptr(), rdo.ctypes.data, rcap.ctypes.data,
                    out.data_ptr(), n, st), "unwrap_async"))
                assert d_dst.cpu().numpy().tobytes() == want, (stages, tag)
                d_dst, (off, out) = torch.zeros(rtotal, dtype=torch.uint8, device="cuda"), outs()
                count(f"unwrap_packed_async/{tag}/{stages}", lambda: native.check(
                    lib.lz4b200_unwrap_batch_packed_to_device_async(
                        h, pk.data_ptr(), pso.ctypes.data, plen.ctypes.data, d_dst.data_ptr(), rtotal, off.data_ptr(),
                        out.data_ptr(), n, st), "unwrap_packed_async"))
                assert d_dst.cpu().numpy().tobytes() == want and int(off[n]) == rtotal, (stages, tag)
    finally:
        ctx.set_option("host_chunk_mb", 128)


def test_gpu_launch_counts_of_every_call_family(ctx):
    count = _Counter(ctx)
    for n in (1, 12):
        _batch_calls(ctx, count, n)
        _framing_calls(ctx, count, n)
    _decoder_calls(ctx, count)
    _placed_calls(ctx, count)
    _async_calls(ctx, count)
    assert count.counts == EXPECTED, "\n" + "\n".join(f"    {k!r}: {v}," for k, v in count.counts.items())


def _prepared(ctx, wrap, n, size, seed):
    """Device inputs and outputs of a packed decode (wrap = False) or a packed unwrap of n entries, and the raw bytes."""
    import torch
    from tests.test_wrap_device_gpu import _host_wrap
    raws = [cases.content(cases.MODELS[(seed + i) % len(cases.MODELS)], size + i % 7, seed=seed + i).tobytes() for i in range(n)]
    buf, so, sl = _src(_host_wrap(ctx, raws, False) if wrap else [oracle.encode(d)[1] for d in raws])
    dst = torch.zeros(sum(len(d) for d in raws), dtype=torch.uint8, device="cuda")
    off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    out = torch.zeros(n, dtype=torch.int32, device="cuda")
    return wrap, (_dev(buf), _dev(so), _dev(sl), dst, off, out), raws


def _enqueue(ctx, prepared):
    from lz4net_b200 import batch
    wrap, args, _ = prepared
    (batch.unwrap_packed if wrap else batch.decode_packed)(ctx, *args)


def _check(prepared):
    _, (_, _, _, dst, off, out), raws = prepared
    sizes = [len(d) for d in raws]
    assert out.cpu().tolist() == sizes
    assert off.cpu().tolist() == np.concatenate([[0], np.cumsum(sizes)]).tolist()
    assert dst.cpu().numpy().tobytes() == b"".join(raws)


@pytest.mark.parametrize("second_grows", [True, False], ids=["second-grows-the-scratch", "scratch-already-large-enough"])
def test_gpu_call_scratch_is_shared_safely_across_streams(ctx, second_grows):
    """Two packed unwraps share the context's call scratch (scan scratch, capacities, packet view) on two torch streams,
    with no synchronise in between: first a small one (40 packets of 2 MiB, whose decode runs long), then a large one
    (6000 packets) held back on its own stream so that, were the two not ordered, its prep would rewrite the small call's
    packet view while the small call's decode and finish still read it.  Either the large call grows the scratch, behind
    a cudaDeviceSynchronize, or an earlier large call already grew it: then nothing grows and only the large call's wait
    on the small call's compact_done keeps them apart."""
    import torch
    small = _prepared(ctx, True, 40, 2 << 20, 7)
    large = _prepared(ctx, True, 6000, 32768, 11)
    if not second_grows:
        _enqueue(ctx, large)
        torch.cuda.synchronize()
        _check(large)
        for t in large[1][3:]:
            t.zero_()
    torch.cuda.synchronize()
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(a):
        _enqueue(ctx, small)
    with torch.cuda.stream(b):
        torch.cuda._sleep(200_000)                        # ~0.1 ms: inside the small call's decode
        _enqueue(ctx, large)
    torch.cuda.synchronize()
    _check(small)
    _check(large)
