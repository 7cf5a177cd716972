"""The LZ4HC kernels on the H100 on the constructed blocks of tests/hcedge.py: the catalogue as one batch under every
kernel choice and under the launch options that select other instantiations and slot counts, a device-memory batch at
every source and destination alignment, capacity sweeps and the block r93 gives up on at LZ4_compressBound.  Every
result and every byte equals the oracle's and the reference's digest in tests/golden/hc_constructed_v1.json."""
import contextlib
import hashlib
import json
import os

import numpy as np
import pytest

import oracle
from tests import hcedge

pytestmark = pytest.mark.gpu

GUARD = 64
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "hc_constructed_v1.json")


@pytest.fixture(scope="module")
def ctx():
    import lz4net_b200
    return lz4net_b200.default_context()


@pytest.fixture(scope="module")
def catalogue():
    return hcedge.catalogue(1)


@pytest.fixture(scope="module")
def golden():
    return {row[0]: row for row in json.load(open(GOLDEN))["cases"]}


@contextlib.contextmanager
def _options(ctx, **opts):
    prev = {k: ctx.get_option(k) for k in opts}
    try:
        for k, v in opts.items():
            ctx.set_option(k, v)
        yield
    finally:
        for k, v in prev.items():
            ctx.set_option(k, v)


def _encode_host(ctx, blocks, caps):
    """One host-memory HC batch, every output slot followed by GUARD bytes that must stay untouched."""
    n = len(blocks)
    lens = np.array([len(b) for b in blocks], np.int32)
    src = np.frombuffer(b"".join(blocks) + b"\0", np.uint8)
    src_off = np.concatenate([[0], np.cumsum(lens[:-1], dtype=np.int64)]).astype(np.int64)
    caps = np.array(caps, np.int32)
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


def _check(catalogue, golden, got, what):
    for c, (r, o) in zip(catalogue, got):
        g = golden[c.name]
        assert (r, o) == oracle.encode_hc(c.data), (c.name, what)
        assert (r, hashlib.sha256(o).hexdigest()) == (g[1], g[2]), (c.name, what)


CONFIGS = [dict(hc_kernel=-1), dict(hc_kernel=0), dict(hc_kernel=1), dict(hc_kernel=2),
           dict(hc_kernel=1, hc_warps_per_sm=1), dict(hc_kernel=1, hc_warps_per_sm=2),
           dict(hc_kernel=2, hc_warps_per_sm=8), dict(hc_kernel=2, hc_warps_per_sm=16),
           dict(hc_kernel=2, hc_warps_per_sm=17),
           dict(hc_kernel=0, hc_concurrency=32), dict(hc_kernel=0, hc_concurrency=33)]


@pytest.mark.parametrize("opts", CONFIGS, ids=lambda o: "-".join(f"{k[3:]}{v}" for k, v in o.items()))
def test_catalogue_as_one_batch(ctx, catalogue, golden, opts):
    """hc_warps_per_sm up to 16 runs the read-through-L1 kernel's 16-warp instantiation, 17 the 32-warp one; 1 and 2 give
    the shared-memory kernel's blocks a larger share of the SM; hc_concurrency below the batch's size reuses the thread
    kernel's slots."""
    with _options(ctx, **opts):
        got = _encode_host(ctx, [c.data for c in catalogue], [oracle.bound(len(c.data)) for c in catalogue])
    _check(catalogue, golden, got, opts)


@pytest.mark.parametrize("hc_kernel", [0, 1, 2])
def test_device_batch_at_every_alignment(ctx, catalogue, golden, hc_kernel):
    """The catalogue in device memory, block i at source offset i % 16 and destination offset 7 i % 16 from a 16-byte
    boundary, GUARD bytes behind every slot."""
    import torch
    n = len(catalogue)
    blocks = [c.data for c in catalogue]
    src_off, dst_off, pos = [], [], 0
    for i, b in enumerate(blocks):
        pos = (pos + 15) // 16 * 16 + i % 16
        src_off.append(pos); pos += len(b)
    src = np.zeros(pos + 16, np.uint8)
    for o, b in zip(src_off, blocks):
        src[o:o + len(b)] = np.frombuffer(b, np.uint8)
    caps = [oracle.bound(len(b)) for b in blocks]
    pos = 0
    for i, c in enumerate(caps):
        pos = (pos + 15) // 16 * 16 + (7 * i) % 16
        dst_off.append(pos); pos += c + GUARD
    d_src = torch.tensor(src, device="cuda")
    d_dst = torch.full((pos,), 0xEE, dtype=torch.uint8, device="cuda")
    d_so = torch.tensor(src_off, dtype=torch.int64, device="cuda")
    d_sl = torch.tensor([len(b) for b in blocks], dtype=torch.int32, device="cuda")
    d_do = torch.tensor(dst_off, dtype=torch.int64, device="cuda")
    d_dc = torch.tensor(caps, dtype=torch.int32, device="cuda")
    d_out = torch.zeros(n, dtype=torch.int32, device="cuda")
    with _options(ctx, hc_kernel=hc_kernel):
        ctx.encode_batch_ptr(d_src.data_ptr(), d_so.data_ptr(), d_sl.data_ptr(), d_dst.data_ptr(), d_do.data_ptr(),
                             d_dc.data_ptr(), d_out.data_ptr(), n, hc=True, device=True)
        torch.cuda.synchronize()
    dst, out = d_dst.cpu().numpy(), d_out.cpu().numpy()
    got = []
    for i in range(n):
        o, c, r = dst_off[i], caps[i], int(out[i])
        assert (dst[o + max(r, 0): o + c + GUARD] == 0xEE).all(), f"block {i}: bytes written behind out_len"
        got.append((r, dst[o:o + max(r, 0)].tobytes()))
    _check(catalogue, golden, got, hc_kernel)


@pytest.mark.parametrize("hc_kernel", [0, 1, 2])
def test_capacity_sweeps(ctx, catalogue, golden, hc_kernel):
    """Every capacity from 0 to past the compressed size over a small block, and the capacities around the start, the
    middle and the end of the output over a window block, as one batch each; cap = n and cap = ret - 1 over the whole
    catalogue against the reference's digests."""
    by = {c.name: c.data for c in catalogue}
    small, win = by["search-budget-repeat-delta4"], by["window-q131072-65535"]
    rs, rw = oracle.encode_hc(small)[0], oracle.encode_hc(win)[0]
    sweeps = [(small, list(range(0, rs + 3))),
              (win, sorted({0, 1, 2, 15, 16, 17, 270, 4096, 65535, 65536, len(win), rw - 3, rw - 2, rw - 1, rw, rw + 1}))]
    with _options(ctx, hc_kernel=hc_kernel):
        for d, caps in sweeps:
            got = _encode_host(ctx, [d] * len(caps), caps)
            for cap, g in zip(caps, got):
                assert g == oracle.encode_hc(d, cap=cap), (hc_kernel, len(d), cap)
        for col, capf in ((3, lambda c, g: len(c.data)), (5, lambda c, g: g[1] - 1)):
            sel = [c for c in catalogue if golden[c.name][1] > 0]
            caps = [capf(c, golden[c.name]) for c in sel]
            got = _encode_host(ctx, [c.data for c in sel], caps)
            for c, (r, o) in zip(sel, got):
                g = golden[c.name]
                assert (r, hashlib.sha256(o).hexdigest()) == (g[col], g[col + 1]), (c.name, hc_kernel, col)


@pytest.mark.parametrize("hc_kernel", [-1, 0, 1, 2])
def test_gives_up_at_the_bound_on_every_kernel(ctx, hc_kernel):
    """The random 64 KiB block on which r93's LZ4HC returns 0 with LZ4_compressBound(n) bytes of room, and encodes with
    4096 more."""
    from lz4net_b200 import synth
    d = synth.make_blocks("E0", 1, 65536, seed=3, first_block=1268)[0].tobytes()
    cap = oracle.bound(len(d))
    with _options(ctx, hc_kernel=hc_kernel):
        got = _encode_host(ctx, [d, d], [cap, cap + 4096])
    assert got[0] == (0, b"") and got[1] == oracle.encode_hc(d, cap=cap + 4096), hc_kernel
