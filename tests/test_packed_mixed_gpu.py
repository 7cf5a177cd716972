"""lz4b200_decode_batch_packed_to_device on an H100: raw LZ4 blocks in host memory whose decoded sizes nobody stored,
decoded back to back into device memory through the host pipeline, the compressed bytes crossing PCIe once.

Offsets, results and bytes must be those of lz4b200_decode_batch_packed on a device copy of the batch, however many
pipeline stages the batch spans and wherever the source lies; a malformed block occupies nothing and disturbs nobody; a
destination too small is reported through out_off[n] with nothing written behind it; the call is ordered behind the work
already queued on the caller's stream, refuses the wrong kind of memory, keeps its device scratch at the size of the
pipeline's stages, and leaves the launches of the existing calls as they were."""
import functools
import hashlib

import numpy as np
import pytest

import oracle
from tests import cases
from tests.test_measure import LONG_LITERAL, OVERFLOW, _corrupt
from tests.test_mixed_memory_gpu import _busy, _dev, _host, _Options, _src, CHUNK_MB_DEFAULT

pytestmark = pytest.mark.gpu

LENS = (0, 1, 12, 13, 4095, 4096, 65535, 65536, 65537, 65546, 200000, 1 << 20)
GUARD = 0xA5
E_ARG = -1
NSLOT = 3                                                                # pipeline depth of the host-memory calls
OFFSET_ZERO = bytes([0x10, 0x61, 0, 0, 0x50]) + b"bbbbb"                # a match at offset 0: rejected by design


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@functools.lru_cache(maxsize=None)
def _corpus():
    """(compressed, raw): every content model at every length, fast-encoded; an HC-encoded copy up to 65 546 bytes."""
    out = []
    for i, m in enumerate(cases.MODELS):
        for n in LENS:
            d = cases.content(m, n, seed=90 + i).tobytes()
            out.append((oracle.encode(d)[1], d))
            if n <= 65546 and (i + n) % 2:
                out.append((oracle.encode_hc(d)[1], d))
    return out


def _malformed():
    bad = _corrupt(90)[0]
    d = cases.content("ETEXT", 70000, seed=3).tobytes()
    c = oracle.encode(d)[1]
    return bad + [OVERFLOW, LONG_LITERAL, OFFSET_ZERO, c[:-1], c[: len(c) // 2], c[:1]]


def _packed(ctx, src, so, sl, room, pad=4096, stream=0):
    """The call on host arrays into the first `room` bytes of a guard-filled device buffer of room + pad bytes.
    Returns (status, out_len, out_off, the whole device buffer as a host array)."""
    import torch
    from lz4net_b200 import native
    n = len(so)
    dst = torch.full((room + pad,), GUARD, dtype=torch.uint8, device="cuda")
    off, out = np.full(n + 1, -7, np.int64), np.full(n, 12345, np.int32)
    rc = native.lib().lz4b200_decode_batch_packed_to_device(ctx.handle, src.ctypes.data, so.ctypes.data, sl.ctypes.data,
                                                            dst.data_ptr(), room, off.ctypes.data, out.ctypes.data, n, stream)
    return rc, out.tolist(), off, dst.cpu().numpy()


def _device_packed(ctx, buf, so, sl, room):
    """lz4b200_decode_batch_packed on a device copy of the same source layout: (out_len, out_off, device buffer)."""
    import torch
    from lz4net_b200 import batch
    n = len(so)
    dst = torch.full((room + 4096,), GUARD, dtype=torch.uint8, device="cuda")
    off = torch.full((n + 1,), -7, dtype=torch.int64, device="cuda")
    out = torch.full((n,), 12345, dtype=torch.int32, device="cuda")
    batch.decode_packed(ctx, _dev(buf), _dev(so), _dev(sl), dst[:room], off, out)
    torch.cuda.synchronize()
    return out.cpu().tolist(), off.cpu().numpy(), dst.cpu().numpy()


def _same_results(got, want, exact):
    """Non-negative results are equal; negative ones are the rejecting decoder's own (equal when the decoder is pinned)."""
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w if exact or w >= 0 else g < 0, (i, g, w)


def _stage_count(sl, chunk_mb):
    """The pipeline's stages for these compressed lengths: blocks are added while the stage stays within chunk_mb."""
    stages, fill = 0, None
    for l in sl:
        if fill is None or fill + int(l) > chunk_mb << 20:
            stages, fill = stages + 1, 0
        fill += int(l)
    return stages


# ---- parity with the device call ------------------------------------------------------------------------------------
@pytest.mark.parametrize("lanes", [0, 16, 1], ids=["auto", "lanes16", "lpb"])
@pytest.mark.parametrize("pinned,chunk_mb", [(False, CHUNK_MB_DEFAULT), (True, CHUNK_MB_DEFAULT), (True, 1), (False, 1)],
                         ids=["pageable-one-stage", "pinned-one-stage", "pinned-many-stages", "pageable-many-stages"])
def test_gpu_packed_from_host_equals_the_device_call(ctx, pinned, chunk_mb, lanes):
    pairs = _corpus()
    comp = [c for c, _ in pairs]
    buf, so, sl = _src(comp, skew=5, gap=3)
    need = sum(len(d) for _, d in pairs)
    with _Options(ctx, **({"decode_lanes": lanes} if lanes else {})):
        want, want_off, want_h = _device_packed(ctx, buf, so, sl, need)
        src = _host(len(buf), 0, pinned)
        src[:] = buf
        with _Options(ctx, host_chunk_mb=chunk_mb):
            rc, got, off, h = _packed(ctx, src, so, sl, need)
    assert rc == 0 and got == want == [len(d) for _, d in pairs]
    assert np.array_equal(off, want_off) and int(off[-1]) == need
    assert h[:need].tobytes() == want_h[:need].tobytes() == b"".join(d for _, d in pairs)
    assert (h[need:] == GUARD).all()
    assert _stage_count(sl, 1) > NSLOT                               # (with 1 MiB stages every slot is used more than once)


def test_gpu_packed_from_host_over_many_stages_and_a_stage_of_one_block(ctx):
    """311 blocks (a prime) over more than NSLOT stages of 1 MiB: incompressible blocks of 1 MiB are a stage each, the rest
    share stages; some blocks are malformed, some empty.  The launches show that the stages ran one by one."""
    blocks, raws = [], []
    for i in range(311):
        m = ("E0", "E50", "ETEXT", "mixed", "E0", "runs", "E100")[i % 7]
        n = 1 << 20 if i % 40 == 7 else (0 if i % 50 == 9 else 20000 + 211 * i)
        d = cases.content(m, n, seed=200 + i).tobytes()
        c = oracle.encode(d)[1]
        if i % 31 == 4:
            c, d = c[: len(c) // 2], None
        blocks.append(c); raws.append(d)
    buf, so, sl = _src(blocks, skew=1, gap=2)
    stages = _stage_count(sl, 1)
    assert stages >= 10 and stages > NSLOT and sum(len(c) > 1 << 20 for c in blocks) >= 3
    want, want_off, want_h = _device_packed(ctx, buf, so, sl, 1)                              # the sizes, from a call that does not fit
    need = int(want_off[-1])
    want, want_off, want_h = _device_packed(ctx, buf, so, sl, need)
    src = _host(len(buf), 0, True)
    src[:] = buf
    with _Options(ctx, host_chunk_mb=1):
        before = ctx.launches
        rc, got, off, h = _packed(ctx, src, so, sl, need)
        launched = ctx.launches - before
    assert rc == 0 and np.array_equal(off, want_off)
    _same_results(got, want, exact=False)
    assert h[:need].tobytes() == want_h[:need].tobytes() and (h[need:] == GUARD).all()
    for i, d in enumerate(raws):
        if d is None:
            assert got[i] < 0 and off[i + 1] == off[i], i
        else:
            assert got[i] == len(d) and h[off[i]:off[i + 1]].tobytes() == d, i
    assert all(oracle.decode_unknown(c, 1 << 21)[0] < 0 for c, d in zip(blocks, raws) if d is None)
    assert launched >= 6 * stages                                    # measure, three scan kernels, placement, a decoder: per stage


# ---- where the source lies --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["pageable", "pinned", "registered"])
@pytest.mark.parametrize("chunk_mb", [1, CHUNK_MB_DEFAULT], ids=["many-stages", "one-stage"])
def test_gpu_packed_from_host_source_placement(ctx, kind, chunk_mb):
    """Pageable, page-locked and lz4b200_host_register'ed sources; blocks in shuffled order with gaps between them; entries
    that share bytes (the same block twice, and a truncated prefix of it)."""
    from lz4net_b200 import native
    pairs = [p for p in _corpus() if len(p[1]) <= 200000]
    comp = [c for c, _ in pairs]
    order = np.random.default_rng(8).permutation(len(comp))
    so = np.zeros(len(comp), np.int64)
    pos = 9
    for i in order:
        so[i] = pos
        pos += len(comp[i]) + 7
    sl = np.array([len(c) for c in comp], np.int32)
    buf = np.zeros(pos + 16, np.uint8)
    for o, c in zip(so, comp):
        buf[o:o + len(c)] = np.frombuffer(c, np.uint8)
    big = max(range(len(comp)), key=lambda i: len(comp[i]))
    so = np.concatenate([so, [so[big], so[big], so[3]]]).astype(np.int64)                     # shared bytes
    sl = np.concatenate([sl, [sl[big], sl[big] // 2, sl[3]]]).astype(np.int32)
    raws = [d for _, d in pairs] + [pairs[big][1], None, pairs[3][1]]
    need = sum(len(d) for d in raws if d is not None)
    src = _host(len(buf), 0, kind == "pinned")
    src[:] = buf
    if kind == "registered":
        native.check(native.lib().lz4b200_host_register(src.ctypes.data, src.nbytes), "host_register")
    try:
        with _Options(ctx, host_chunk_mb=chunk_mb):
            rc, got, off, h = _packed(ctx, src, so, sl, need)
    finally:
        if kind == "registered":
            native.check(native.lib().lz4b200_host_unregister(src.ctypes.data), "host_unregister")
    assert rc == 0 and int(off[-1]) == need and (h[need:] == GUARD).all()
    for i, d in enumerate(raws):
        if d is None:
            assert got[i] < 0 and off[i + 1] == off[i]
        else:
            assert got[i] == len(d) and h[off[i]:off[i + 1]].tobytes() == d, i


# ---- malformed blocks -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk_mb", [1, CHUNK_MB_DEFAULT], ids=["many-stages", "one-stage"])
@pytest.mark.parametrize("lanes", [0, 16], ids=["auto", "lanes16"])
def test_gpu_packed_from_host_malformed_blocks_occupy_nothing(ctx, lanes, chunk_mb):
    """Truncated, bit-flipped, length-overflow and offset-0 blocks between well-formed ones: a negative out_len, no bytes, the
    neighbours bit-exact and back to back -- so every byte of the destination is accounted for by a well-formed block, and
    nothing behind the total changes."""
    good = [p for p in _corpus() if 0 < len(p[1]) <= 65546][:60]
    bad = _malformed()
    blocks, raws = [], []
    for i in range(max(len(good), len(bad))):
        if i < len(bad):
            blocks.append(bad[i]); raws.append(None)
        if i < len(good):
            blocks.append(good[i][0]); raws.append(good[i][1])
    blocks += [b"", b""]; raws += [None, None]                                                 # an empty stream is malformed too
    buf, so, sl = _src(blocks, skew=5, gap=3)
    with _Options(ctx, **({"decode_lanes": lanes} if lanes else {})):
        want, want_off, _ = _device_packed(ctx, buf, so, sl, 1)
        need = int(want_off[-1])
        want, want_off, want_h = _device_packed(ctx, buf, so, sl, need)
        with _Options(ctx, host_chunk_mb=chunk_mb):
            rc, got, off, h = _packed(ctx, buf, so, sl, need)
    assert rc == 0 and np.array_equal(off, want_off)
    _same_results(got, want, exact=bool(lanes))
    assert h[:need].tobytes() == want_h[:need].tobytes() and (h[need:] == GUARD).all()
    for i, d in enumerate(raws):
        if d is not None:
            assert got[i] == len(d) and h[off[i]:off[i + 1]].tobytes() == d, i
        elif want[i] < 0:                                            # (a bit flip may leave a stream the format accepts)
            assert got[i] < 0 and off[i + 1] == off[i], i
    assert got[blocks.index(OFFSET_ZERO)] < 0 and got[blocks.index(OVERFLOW)] < 0 and got[-1] < 0
    assert sum(g < 0 for g in got) > 30


# ---- a destination that is too small ----------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk_mb", [1, CHUNK_MB_DEFAULT], ids=["many-stages", "one-stage"])
def test_gpu_packed_from_host_that_does_not_fit(ctx, chunk_mb):
    """total - 1, half and 0 bytes of room: LZ4B200_OK, out_off as if it had fitted, out_len = the sizes for well-formed
    blocks and negative for the others, nothing written behind the room; then exactly the total fits."""
    pairs = [p for p in _corpus() if len(p[1]) <= 200000]
    blocks = [c for c, _ in pairs] + _malformed()
    order = np.random.default_rng(4).permutation(len(blocks))
    blocks = [blocks[i] for i in order]
    buf, so, sl = _src(blocks, skew=2, gap=1)
    sizes, _, _ = _device_packed(ctx, buf, so, sl, 1)
    want_off = np.concatenate([[0], np.cumsum(np.maximum(sizes, 0), dtype=np.int64)])
    need = int(want_off[-1])
    with _Options(ctx, host_chunk_mb=chunk_mb):
        for room in (need - 1, need // 2, 0):
            rc, got, off, h = _packed(ctx, buf, so, sl, room)
            assert rc == 0 and np.array_equal(off, want_off), room
            _same_results(got, sizes, exact=False)
            assert (h[room:] == GUARD).all(), "a byte behind dst_total_cap changed"
        rc, got, off, h = _packed(ctx, buf, so, sl, need)                                     # the second call, with out_off[n] bytes
    assert rc == 0 and np.array_equal(off, want_off) and (h[need:] == GUARD).all()
    _same_results(got, sizes, exact=False)
    _, _, want_h = _device_packed(ctx, buf, so, sl, need)
    assert h[:need].tobytes() == want_h[:need].tobytes()
    assert sum(s < 0 for s in sizes) > 20 and need > 1 << 20


def test_gpu_packed_from_host_bad_arguments_and_empty_batches(ctx):
    import torch
    from lz4net_b200 import batch, native
    l = native.lib()
    blocks = [oracle.encode(cases.content("E50", 3000 + i, seed=i).tobytes())[1] for i in range(4)]
    buf, so, sl = _src(blocks)
    need = sum(3000 + i for i in range(4))
    d_dst = torch.full((need + 64,), GUARD, dtype=torch.uint8, device="cuda")
    h_dst = np.full(need + 64, 0xEE, np.uint8)
    off, out = np.full(5, -7, np.int64), np.full(4, 12345, np.int32)
    p = lambda a: a.ctypes.data                                                              # noqa: E731
    call = lambda src, dst, sl_=sl, off_=p(off), room=need: l.lz4b200_decode_batch_packed_to_device(   # noqa: E731
        ctx.handle, src, p(so), p(sl_), dst, room, off_, p(out), 4, 0)
    neg = sl.copy(); neg[2] = -1
    assert call(_dev(buf).data_ptr(), d_dst.data_ptr()) == E_ARG                             # device src as the host side
    assert call(p(buf), p(h_dst)) == E_ARG                                                   # host dst as the device side
    assert call(p(buf), d_dst.data_ptr(), sl_=neg) == E_ARG                                  # a negative length
    assert call(p(buf), d_dst.data_ptr(), off_=None) == E_ARG and call(p(buf), d_dst.data_ptr(), room=-1) == E_ARG
    assert call(p(buf), None) == E_ARG
    if torch.cuda.device_count() > 1:
        other = torch.full((need + 64,), GUARD, dtype=torch.uint8, device="cuda:1")
        assert call(p(buf), other.data_ptr()) == E_ARG                                       # another GPU's memory
        assert bool((other == GUARD).all())
    torch.cuda.synchronize()
    assert bool((d_dst == GUARD).all()) and (h_dst == 0xEE).all() and (off == -7).all() and (out == 12345).all(), \
        "a refused call wrote something"
    assert call(p(buf), d_dst.data_ptr()) == 0 and out.tolist() == [3000, 3001, 3002, 3003] and off[4] == need
    z = np.full(1, -7, np.int64)
    assert l.lz4b200_decode_batch_packed_to_device(ctx.handle, None, None, None, None, 0, p(z), None, 0, 0) == 0 and z[0] == 0
    e64, e32 = np.zeros(0, np.int64), np.zeros(0, np.int32)
    z[0] = -7
    assert batch.decode_from_host_packed(ctx, buf, e64, e32, d_dst, z, e32) == 0 and z[0] == 0


# ---- ordering behind the caller's stream ------------------------------------------------------------------------------
def test_gpu_packed_from_host_waits_for_readers_of_the_old_contents(ctx):
    """A dst.clone() queued on a non-default stream behind a long kernel chain, then at once a packed decode into dst given
    that stream: the clone holds the old contents, not the decoded bytes."""
    import torch
    from lz4net_b200 import batch
    raws = [cases.content("ETEXT", 65536, seed=i).tobytes() for i in range(64)]
    buf, so, sl = _src([oracle.encode(d)[1] for d in raws])
    dst = torch.full((64 * 65536,), 0x5A, dtype=torch.uint8, device="cuda")
    off, res = np.zeros(65, np.int64), np.zeros(64, np.int32)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    _busy(s)
    with torch.cuda.stream(s), _Options(ctx, host_chunk_mb=1):
        snap = dst.clone()
        total = batch.decode_from_host_packed(ctx, buf, so, sl, dst, off, res)
    s.synchronize()
    assert bool((snap == 0x5A).all()), "the decode overwrote dst before an earlier reader on the stream was done"
    assert total == 64 * 65536 and res.tolist() == [65536] * 64 and dst.cpu().numpy().tobytes() == b"".join(raws)


# ---- large batches ----------------------------------------------------------------------------------------------------
def _encoded_on_device(ctx, cls, nb, bs, seed):
    """nb synthetic blocks encoded on the device and packed into host memory: (sha256 of the raw bytes, packed, off, len)."""
    import torch
    from lz4net_b200 import batch, synth
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    batch.synth_fill(ctx, raw, nb, bs, synth.CLASS_ID[cls], seed=seed)
    so = np.arange(nb, dtype=np.int64) * bs
    sl = np.full(nb, bs, np.int32)
    caps = np.full(nb, oracle.bound(bs), np.int32)
    packed = torch.empty(nb * int(caps[0]), dtype=torch.uint8).pin_memory().numpy()
    off, clen = np.zeros(nb + 1, np.int64), np.zeros(nb, np.int32)
    batch.encode_to_host_packed(ctx, raw, so, sl, caps, packed, off, clen)
    return hashlib.sha256(raw.cpu().numpy().tobytes()).hexdigest(), packed, off[:-1].copy(), clen


@pytest.mark.parametrize("cls", ["E0", "E50", "E100", "ETEXT"])
def test_gpu_packed_from_host_large_synthetic_batch(ctx, cls):
    """2^13 x 64 KiB blocks of each entropy class at the default stage size: the decoded bytes hash like the source."""
    import torch
    from lz4net_b200 import batch
    nb, bs = 1 << 13, 65536
    digest, packed, so, sl = _encoded_on_device(ctx, cls, nb, bs, seed=41)
    out = torch.zeros(nb * bs, dtype=torch.uint8, device="cuda")
    off, res = np.zeros(nb + 1, np.int64), np.zeros(nb, np.int32)
    assert batch.decode_from_host_packed(ctx, packed, so, sl, out, off, res) == nb * bs
    assert (res == bs).all() and np.array_equal(off, np.arange(nb + 1, dtype=np.int64) * bs)
    assert hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest() == digest


def test_gpu_packed_from_host_device_memory_is_flat_in_the_batch_size(ctx):
    """The device memory a fresh context adds for the packed decode of 256 MiB and of 1 GiB of E50 differs by less than one
    pipeline stage, and stays far below the batch.  (32 MiB stages: both batches keep all three slots full.)"""
    import torch
    import lz4net_b200
    from lz4net_b200 import batch
    bs, stage_mb = 65536, 32
    added = {}
    for mib in (256, 1024):
        nb = (mib << 20) // bs
        _, packed, so, sl = _encoded_on_device(ctx, "E50", nb, bs, seed=mib)
        out = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
        off, res = np.zeros(nb + 1, np.int64), np.zeros(nb, np.int32)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        free0 = torch.cuda.mem_get_info()[0]
        c = lz4net_b200.Context(0)
        c.set_option("host_chunk_mb", stage_mb)
        assert batch.decode_from_host_packed(c, packed, so, sl, out, off, res) == nb * bs
        torch.cuda.synchronize()
        added[mib] = free0 - torch.cuda.mem_get_info()[0]
        c.close()
        assert (res == bs).all()
        del out
        torch.cuda.empty_cache()
    assert abs(added[1024] - added[256]) < stage_mb << 20, added
    assert added[1024] < 256 << 20, added


# ---- the existing calls ----------------------------------------------------------------------------------------------
def test_gpu_existing_calls_enqueue_the_launches_they_did(ctx):
    """64 ETEXT blocks of 64 KiB, the decoder picked automatically: lz4b200_decode_batch_packed is 10 launches (measure, three
    scan kernels, placement, the counters' reset, the pick and its candidates), lz4b200_unwrap_batch_packed 11 (the header
    prep in place of the measure, and the finish), a LZ4B200_MEM_HOST_TO_DEVICE known-size decode of one stage 1 (the
    counters' reset is what a decode with a decoder chosen on the host counts) -- as before the placement kernel learnt to
    carry a running offset."""
    import torch
    from lz4net_b200 import batch
    from tests.test_wrap_device_gpu import _host_wrap
    raws = [cases.content("ETEXT", 65536, seed=i).tobytes() for i in range(64)]
    comp = [oracle.encode(d)[1] for d in raws]
    buf, so, sl = _src(comp)
    need = 64 * 65536
    dst = torch.zeros(need, dtype=torch.uint8, device="cuda")
    off = torch.zeros(65, dtype=torch.int64, device="cuda")
    out = torch.zeros(64, dtype=torch.int32, device="cuda")
    d_buf, d_so, d_sl = _dev(buf), _dev(so), _dev(sl)
    before = ctx.launches
    batch.decode_packed(ctx, d_buf, d_so, d_sl, dst, off, out)
    torch.cuda.synchronize()
    assert ctx.launches - before == 10 and out.cpu().tolist() == [65536] * 64
    pbuf, pso, psl = _src(_host_wrap(ctx, raws, False))
    d_buf, d_so, d_sl = _dev(pbuf), _dev(pso), _dev(psl)
    before = ctx.launches
    batch.unwrap_packed(ctx, d_buf, d_so, d_sl, dst, off, out)
    torch.cuda.synchronize()
    assert ctx.launches - before == 11 and out.cpu().tolist() == [65536] * 64
    res = np.zeros(64, np.int32)
    do, caps = np.arange(64, dtype=np.int64) * 65536, np.full(64, 65536, np.int32)
    before = ctx.launches
    batch.decode_from_host(ctx, buf, so, sl, dst, do, caps, res)
    assert ctx.launches - before == 1 and res.tolist() == [len(c) for c in comp]
    assert dst.cpu().numpy().tobytes() == b"".join(raws)


# ---- the Python surface ----------------------------------------------------------------------------------------------
def test_gpu_context_decode_blocks_to_device_and_lz4codec_decode_into_a_tensor(ctx):
    import torch
    from lz4net_b200 import LZ4Codec
    raws = [cases.content(m, n, seed=7).tobytes() for m, n in (("ETEXT", 100000), ("E100", 5000), ("runs", 13), ("E50", 0))]
    comp = [LZ4Codec.Encode(d) if d else b"" for d in raws]
    need = sum(len(d) for d in raws)
    out = torch.full((need + 64,), GUARD, dtype=torch.uint8, device="cuda")
    res, off = ctx.decode_blocks_to_device(comp + [OFFSET_ZERO], out[:need])
    assert res[:3] == [len(d) for d in raws[:3]] and res[3] < 0 and res[4] < 0                 # an empty stream is malformed
    assert off == [0, 100000, 105000, 105013, 105013, 105013]
    h = out.cpu().numpy()
    assert h[:need].tobytes() == b"".join(raws) and (h[need:] == GUARD).all()
    res, off = ctx.decode_blocks_to_device(comp, out[:100])                                  # too small: the sizes
    assert off[-1] == need and res[:3] == [100000, 5000, 13]
    assert ctx.decode_blocks_to_device([], out) == ([], [0])
    # LZ4Codec.Decode(..., knownOutputLength=False) into a tensor's bytes: offset and length count bytes
    f = torch.zeros(30000, dtype=torch.float32, device="cuda")
    assert LZ4Codec.Decode(comp[0], 0, len(comp[0]), f, 16, 110000, False) == 100000
    assert f.view(torch.uint8)[16:100016].cpu().numpy().tobytes() == raws[0]
    assert not bool(f.view(torch.uint8)[:16].any()) and not bool(f.view(torch.uint8)[100016:].any())
    assert LZ4Codec.Decode(comp[0], 0, 0, f, 0, 100, False) == 0 and LZ4Codec.Decode(comp[0], 0, -1, f, 0, 0, False) == 0
    with pytest.raises(ValueError):
        LZ4Codec.Decode(comp[0], 0, len(comp[0]), f, 0, 99999, False)                        # one byte short
    with pytest.raises(ValueError):
        LZ4Codec.Decode(comp[0], 0, len(comp[0]) - 1, f, 0, 120000, False)                   # truncated
    with pytest.raises(ValueError):
        LZ4Codec.Decode(OFFSET_ZERO, 0, len(OFFSET_ZERO), f, 0, 120000, False)
    with pytest.raises(TypeError):
        LZ4Codec.Decode(comp[0], 0, len(comp[0]), f, 0, 100000, True)
    with pytest.raises(ValueError):
        LZ4Codec.Decode(comp[0], 0, len(comp[0]), f, 100, 120000, False)                     # offset + length beyond the tensor
