"""LZ4HC blocks above 64 KiB on the GPU: a warp per block over a sliding 64 KiB window (lz4hc_window.cuh), behind the warp
kernel for blocks <= 64 KiB and ahead of the thread kernel, through the C ABI.  Every result is the reference's."""
import numpy as np
import pytest

import oracle
from tests import cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@pytest.fixture(params=[-1, 0, 1, 2], ids=["hc-auto", "hc-thread", "hc-warp-smem", "hc-warp-l1"])
def hck(ctx, request):
    prev = ctx.get_option("hc_kernel")
    ctx.set_option("hc_kernel", request.param)
    yield request.param
    ctx.set_option("hc_kernel", prev)


GUARD = 64


def _encode_host_guarded(ctx, blocks):
    """One host-memory HC batch, every output slot followed by GUARD bytes that must stay untouched."""
    n = len(blocks)
    lens = np.array([len(b) for b in blocks], np.int32)
    src = np.frombuffer(b"".join(blocks) + b"\0", np.uint8)
    src_off = np.concatenate([[0], np.cumsum(lens[:-1], dtype=np.int64)]).astype(np.int64)
    caps = np.array([oracle.bound(int(l)) for l in lens], np.int32)
    dst_off = np.concatenate([[0], np.cumsum(caps.astype(np.int64) + GUARD)[:-1]]).astype(np.int64)
    dst = np.full(int(dst_off[-1] + caps[-1] + GUARD), 0xEE, np.uint8)
    out = np.zeros(n, np.int32)
    ctx.encode_batch_ptr(src.ctypes.data, src_off.ctypes.data, lens.ctypes.data, dst.ctypes.data, dst_off.ctypes.data,
                         caps.ctypes.data, out.ctypes.data, n, hc=True, device=False)
    res = []
    for i in range(n):
        o, c, r = int(dst_off[i]), int(caps[i]), int(out[i])
        assert (dst[o + max(r, 0): o + c + GUARD] == 0xEE).all(), f"block {i}: bytes written behind out_len"
        res.append((r, dst[o:o + max(r, 0)].tobytes()))
    return res


def test_hc_window_mixed_batch(ctx, hck):
    blocks = []
    for i, m in enumerate(cases.MODELS):
        for n in (65536, 65537, 131072, 1 << 20, 4 << 20):
            blocks.append(cases.content(m, n, seed=300 + 7 * i + n % 13).tobytes())
    got = _encode_host_guarded(ctx, blocks)
    for i, (b, g) in enumerate(zip(blocks, got)):
        assert g == oracle.encode_hc(b), (hck, i, len(b))


def test_hc_window_large_device_batch(ctx):
    """More blocks above 64 KiB than warps in flight (132 SMs x 16): 5000 x 128 KiB of ETEXT on the device."""
    import torch
    from lz4net_b200 import batch
    nb, bs = 5000, 131072
    slot = oracle.bound(bs)
    raw = torch.empty(nb * bs, dtype=torch.uint8, device="cuda")
    batch.synth_fill(ctx, raw, nb * 2, 65536, 3, seed=9, first_block=0)
    so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
    slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    batch.encode(ctx, raw, so, sl, slots, do, dc, clen, hc=True)
    torch.cuda.synchronize()
    h_len = clen.cpu().numpy()
    assert (h_len > 0).all()
    for i in list(range(0, nb, 313)) + [nb - 1]:
        r, o = oracle.encode_hc(raw[i * bs:(i + 1) * bs].cpu().numpy().tobytes())
        assert h_len[i] == r and slots[i * slot:i * slot + r].cpu().numpy().tobytes() == o, i


def test_hc_window_single_block_entry_points(ctx):
    from lz4net_b200 import LZ4Codec
    from tests.test_stream_host_logic import _varint
    for n in (300_000, 1 << 20):
        d = cases.content("mixed", n, seed=n).tobytes()
        r, o = oracle.encode_hc(d)
        assert LZ4Codec.EncodeHC(d) == o, n
    d = cases.content("ETEXT", 1 << 20, seed=2).tobytes()
    w = LZ4Codec.WrapHC(d)
    assert LZ4Codec.Unwrap(w) == d
    r, o = oracle.encode_hc(d)
    assert o in w and len(w) - len(o) <= 16
    data = b"".join(cases.content(m, 1 << 20, seed=40 + i).tobytes() for i, m in enumerate(cases.MODELS))
    want = bytearray()                               # LZ4Stream's chunks: flags (1 compressed | 2 high compression), lengths, bytes
    for o in range(0, len(data), 1 << 20):
        blk = data[o:o + (1 << 20)]
        r, c = oracle.encode_hc(blk, cap=len(blk))
        want += _varint(2) + _varint(len(blk)) + blk if r <= 0 or r >= len(blk) else _varint(3) + _varint(len(blk)) + _varint(r) + c[:r]
    assert ctx.stream_encode(data, 1 << 20, high_compression=True) == bytes(want)


def test_hc_window_edge_cases(ctx):
    import torch
    from lz4net_b200 import batch
    # n = 0: nothing to do, no pointer looked at
    ctx.encode_batch_ptr(0, 0, 0, 0, 0, 0, 0, 0, hc=True, device=True)
    # a non-default stream, a device batch of blocks above 64 KiB
    nb, bs = 40, 200_000
    blocks = [cases.content(cases.MODELS[i % 8], bs, seed=i).tobytes() for i in range(nb)]
    raw = torch.tensor(np.frombuffer(b"".join(blocks), np.uint8), device="cuda")
    slot = oracle.bound(bs)
    so, do, sl, dc = batch.uniform_layout(nb, bs, slot, "cuda")
    slots = torch.empty(nb * slot, dtype=torch.uint8, device="cuda")
    clen = torch.zeros(nb, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        batch.encode(ctx, raw, so, sl, slots, do, dc, clen, hc=True)
    s.synchronize()
    for i in range(nb):
        r, o = oracle.encode_hc(blocks[i])
        assert int(clen[i]) == r and slots[i * slot:i * slot + r].cpu().numpy().tobytes() == o, i
    # a batch where every block hands back (the colliding period-3 run, past 64 KiB): the thread kernel encodes it
    from tests import hcedge
    found = hcedge.colliding_triple()
    rng = np.random.default_rng(5)
    back = [rng.integers(0, 256, 70000 + 1000 * i, dtype=np.uint8).tobytes() + bytes(found) * 200 + bytes(300) for i in range(6)]
    lens, outs = ctx.encode_blocks(back, hc=True)
    for b, r, o in zip(back, lens, outs):
        assert (r, o) == oracle.encode_hc(b)
