"""Multi-GPU sharding of a batch of independent blocks (SURVEY.md 8e).

lz4net's blocks are independent by construction (doc/compatibility.md:4-7), so the multi-GPU form of the path is plain
data parallelism: rank r owns the contiguous block range [r*B, (r+1)*B) (weak scaling: B blocks per GPU) or an even
split of a fixed total (strong scaling, used by LZ4Stream-style callers to keep stream order on gather).  The codec has
no data-path collective; bench.py only uses torch.distributed for the barrier and the max-over-ranks of the timings.
When the data starts on one rank (BASELINE configs[3]: one stream, many GPUs) the second half of this module scatters
the blocks from the root and gathers the payloads back, in stream order.
"""
from __future__ import annotations

from typing import Sequence, Tuple


def weak_range(rank: int, blocks_per_rank: int) -> Tuple[int, int]:
    """Global block indices owned by `rank` when every rank processes `blocks_per_rank` blocks."""
    return rank * blocks_per_rank, (rank + 1) * blocks_per_rank


def strong_range(rank: int, world: int, total_blocks: int) -> Tuple[int, int]:
    """Contiguous, order-preserving split of `total_blocks` over `world` ranks (sizes differ by at most one)."""
    base, rem = divmod(total_blocks, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def reduce_max(values: Sequence[float], device=None):
    """Max over ranks of each value (device timings: the slowest rank defines the job's time)."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return [float(v) for v in values]
    t = torch.tensor(list(values), dtype=torch.float64, device=device or "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return [float(x) for x in t.tolist()]


def reduce_sum(values: Sequence[float], device=None):
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return [float(v) for v in values]
    t = torch.tensor(list(values), dtype=torch.float64, device=device or "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return [float(x) for x in t.tolist()]


def aggregate_throughput(bytes_per_rank: float, seconds_this_rank: float, device=None) -> float:
    """Whole-job bytes/s: all ranks' bytes over the slowest rank's time."""
    total = reduce_sum([bytes_per_rank], device)[0]
    worst = reduce_max([seconds_this_rank], device)[0]
    return total / worst


# ----------------------------------------------------------------------------------------------------------------------
# One stream, many GPUs (BASELINE configs[3]): the root rank holds a raw stream chunked into independent blocks; every
# rank encodes a contiguous, order-preserving range of them; the root ends up with every block's compressed length
# and the packed payloads in stream order (exactly what LZ4Stream's writer consumes, src/LZ4/LZ4Stream.cs:239-269).
# The decode direction is the mirror image.  The only exchange steps are the scatter of the inputs and the gather of the
# outputs (point-to-point sends between the root and each peer: NCCL over NVLink on a GPU box, gloo in the CPU tests);
# the codec itself never communicates.  `encode_local` / `decode_local` are the per-rank codec calls -- the GPU batch
# functions below in production, a toy codec in the CPU tests of the plumbing.
# ----------------------------------------------------------------------------------------------------------------------
def _p2p(ops):
    import torch.distributed as dist
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()


def scatter_ranges(root_buf, byte_ranges, rank: int, root: int = 0, like=None):
    """The root sends bytes [lo, hi) of `root_buf` to rank r for byte_ranges[r] = (lo, hi); returns this rank's bytes
    (a view on the root, a new tensor elsewhere).  Every rank passes the same byte_ranges."""
    import torch
    import torch.distributed as dist
    lo, hi = byte_ranges[rank]
    if rank == root:
        _p2p([dist.P2POp(dist.isend, root_buf[a:b], r) for r, (a, b) in enumerate(byte_ranges) if r != root and b > a])
        return root_buf[lo:hi]
    mine = torch.empty(hi - lo, dtype=torch.uint8, device=like.device if like is not None else "cpu")
    _p2p([dist.P2POp(dist.irecv, mine, root)] if hi > lo else [])
    return mine


def gather_ranges(local, byte_ranges, rank: int, root: int = 0, out=None):
    """Mirror of scatter_ranges: rank r's `local` bytes land at byte_ranges[r] of `out` on the root (returned there)."""
    import torch.distributed as dist
    if rank == root:
        lo, hi = byte_ranges[root]
        out[lo:hi] = local[: hi - lo]
        _p2p([dist.P2POp(dist.irecv, out[a:b], r) for r, (a, b) in enumerate(byte_ranges) if r != root and b > a])
        return out
    lo, hi = byte_ranges[rank]
    _p2p([dist.P2POp(dist.isend, local[: hi - lo], root)] if hi > lo else [])
    return None


def _all_gather_i64(value: int, device):
    import torch
    import torch.distributed as dist
    world = dist.get_world_size()
    mine = torch.tensor([int(value)], dtype=torch.int64, device=device)
    out = [torch.zeros(1, dtype=torch.int64, device=device) for _ in range(world)]
    dist.all_gather(out, mine)
    return [int(t.item()) for t in out]


def _post(op, tensor, peer):
    """One point-to-point transfer as its own group (its own kernel on the communicator's stream, so transfers posted one
    after the other run one after the other); returns the work handles."""
    import torch.distributed as dist
    return dist.batch_isend_irecv([dist.P2POp(op, tensor, peer)])


def _wait(works):
    for w in works:
        w.wait()


def encode_stream_sharded(raw_root, n_blocks: int, block_size: int, encode_local, rank: int, world: int, root: int = 0,
                          device=None, pieces: int = 1):
    """raw_root: uint8[n_blocks * block_size] on the root (ignored elsewhere; the last block may not be short).
    encode_local(shard_bytes, m_blocks) -> (packed uint8[...], lens int32[m_blocks]) for m_blocks blocks.
    Returns on the root (lens int32[n_blocks], offsets int64[n_blocks + 1], packed uint8[total]) in stream order,
    (None, None, None) elsewhere.

    Every rank's block range can be cut into `pieces` sub-ranges (all transfers posted up front, a piece encoded as soon
    as it has arrived).  That bought nothing when measured (tools/stream_ab.py): a point-to-point transfer is a
    KERNEL of the communication library, and it is not scheduled while the persistent encode kernel holds every SM's
    shared memory -- the pieces arrive back to back before the first encode or after the last one.  (Sending rank 1 its
    range first, then rank 2's, ... is worse for the same reason.)  The transfers that
    do overlap the kernels are the copy engines' -- StreamWindow below."""
    import torch
    import torch.distributed as dist
    dev = device if device is not None else (raw_root.device if raw_root is not None else "cpu")
    blk = [strong_range(r, world, n_blocks) for r in range(world)]
    like = torch.empty(0, dtype=torch.uint8, device=dev)
    a, b = blk[rank]
    m = b - a
    pieces = max(1, min(pieces, m)) if m else 1
    def sub(r, p, k):                                           # block sub-range p of k of rank r
        lo, hi = blk[r]; n = hi - lo
        return lo + n * p // k, lo + n * (p + 1) // k
    works, bufs = [], []
    for p in range(pieces):
        if rank == root:
            ops = []
            for r in range(world):
                if r == root:
                    continue
                k = max(1, min(pieces, blk[r][1] - blk[r][0])) if blk[r][1] > blk[r][0] else 1
                if p < k:
                    lo, hi = sub(r, p, k)
                    if hi > lo:
                        ops.append(dist.P2POp(dist.isend, raw_root[lo * block_size: hi * block_size], r))
            works.append(dist.batch_isend_irecv(ops) if ops else [])
            lo, hi = sub(root, p, pieces) if m else (0, 0)
            bufs.append(raw_root[lo * block_size: hi * block_size])
        else:
            lo, hi = sub(rank, p, pieces) if m else (0, 0)
            buf = torch.empty((hi - lo) * block_size, dtype=torch.uint8, device=dev)
            works.append(dist.batch_isend_irecv([dist.P2POp(dist.irecv, buf, root)]) if hi > lo else [])
            bufs.append(buf)
    packed_parts, lens_parts = [], []
    for p in range(pieces):
        if rank != root:
            for w in works[p]:
                w.wait()
        lo, hi = sub(rank, p, pieces) if m else (0, 0)
        if hi > lo:
            pk, ln = encode_local(bufs[p], hi - lo)
            packed_parts.append(pk); lens_parts.append(ln)
    if rank == root:
        for ws in works:
            for w in ws:
                w.wait()
    packed = torch.cat(packed_parts) if len(packed_parts) > 1 else (packed_parts[0] if packed_parts else like)
    lens = torch.cat(lens_parts) if len(lens_parts) > 1 else (lens_parts[0] if lens_parts else torch.empty(0, dtype=torch.int32, device=dev))
    total = int(lens.to(torch.int64).sum().item()) if m else 0
    totals = _all_gather_i64(total, dev)                        # every rank's payload size: the only metadata exchanged
    pay = [(sum(totals[:r]), sum(totals[:r + 1])) for r in range(world)]
    out = torch.empty(sum(totals), dtype=torch.uint8, device=dev) if rank == root else None
    out = gather_ranges(packed, pay, rank, root, out)
    lens_all = torch.empty(n_blocks * 4, dtype=torch.uint8, device=dev) if rank == root else None
    lens_all = gather_ranges(lens.contiguous().view(torch.uint8) if m else like, [(x * 4, y * 4) for x, y in blk], rank, root, lens_all)
    if rank != root:
        return None, None, None
    lens_i = lens_all.view(torch.int32)
    off = torch.zeros(n_blocks + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(lens_i.to(torch.int64), 0)
    return lens_i, off, out


def decode_stream_sharded(packed_root, lens_root, n_blocks: int, block_size: int, decode_local, rank: int, world: int,
                          root: int = 0, device=None):
    """Mirror image: packed_root / lens_root (int32[n_blocks]) on the root; decode_local(packed, lens, m_blocks, out=None)
    -> uint8[m_blocks * block_size] (written into `out` when given).  Returns the raw stream on the root, None elsewhere.
    Staggered like the encode: rank r gets its lengths and its payload before rank r+1 does, and its decoded blocks cross
    back (the root's ingress: the long leg) while the later ranks still receive and decode."""
    import torch
    import torch.distributed as dist
    dev = device if device is not None else (packed_root.device if packed_root is not None else "cpu")
    blk = [strong_range(r, world, n_blocks) for r in range(world)]
    a, b = blk[rank]
    m = b - a
    if rank != root:
        if m:
            lens = torch.empty(m, dtype=torch.int32, device=dev)
            _wait(_post(dist.irecv, lens, root))
            mine = torch.empty(int(lens.to(torch.int64).sum().item()), dtype=torch.uint8, device=dev)
            _wait(_post(dist.irecv, mine, root))
            raw = decode_local(mine, lens, m)
            _wait(_post(dist.isend, raw, root))
        return None
    lens = lens_root.to(torch.int32).contiguous()
    off = torch.zeros(n_blocks + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(lens.to(torch.int64), 0)
    edges = off[torch.tensor([x for ab in blk for x in ab], dtype=torch.int64, device=dev)].tolist()   # 2 per rank, not n_blocks
    works = []
    for r in range(world):
        lo, hi = blk[r]
        if r != root and hi > lo:
            works += _post(dist.isend, lens[lo:hi], r)
            works += _post(dist.isend, packed_root[edges[2 * r]: edges[2 * r + 1]], r)
    out = torch.empty(n_blocks * block_size, dtype=torch.uint8, device=dev)
    for r in range(world):                                       # posted before the root's own decode: they fill as peers finish
        lo, hi = blk[r]
        if r != root and hi > lo:
            works += _post(dist.irecv, out[lo * block_size: hi * block_size], r)
    if m:
        decode_local(packed_root[edges[2 * root]: edges[2 * root + 1]], lens[a:b], m, out=out[a * block_size: b * block_size])
    _wait(works)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# The same job over peer memory (NVLink 5 / NVSwitch, CUDA IPC): the stream's buffers live in a WINDOW on the root that
# every rank has mapped, and the peers move their ranges themselves with device-to-device copies between the window and
# local buffers.  Those copies run on the copy engines, not on SMs, so -- unlike a send/recv kernel -- they do overlap the
# persistent codec kernels: a rank pulls piece p+1 and pushes piece p-1 while piece p is in the kernel.  The only
# collective is a barrier on either side (plus an all-gather of one payload size per rank on the encode side).
# ----------------------------------------------------------------------------------------------------------------------
class StreamWindow:
    """Root-resident buffers of one stream of n_blocks x block_size bytes, mapped by every rank:
    raw uint8[n_blocks * block_size], packed uint8[n_blocks * bound], lens int32[n_blocks], off int64[n_blocks + 1].
    Created collectively, once (the mapping costs milliseconds: like a communicator, it is set up outside the data path)
    and reused for any number of encode / decode calls.  GPU only (one process per GPU on one node)."""

    def __init__(self, n_blocks: int, block_size: int, rank: int, world: int, root: int = 0, device=None, bound_per_block: int = 0):
        import torch
        import torch.distributed as dist
        from torch.multiprocessing.reductions import reduce_tensor
        self.n_blocks, self.block_size, self.rank, self.world, self.root = n_blocks, block_size, rank, world, root
        self.bound = bound_per_block or (block_size + block_size // 255 + 16)
        self.device = device
        names = ("raw", "packed", "lens", "off")
        handles, err = [None], None
        if rank == root:                                         # a failure on one rank must not leave the others waiting
            try:
                self.raw = torch.empty(n_blocks * block_size, dtype=torch.uint8, device=device)
                self.packed = torch.empty(n_blocks * self.bound, dtype=torch.uint8, device=device)
                self.lens = torch.zeros(n_blocks, dtype=torch.int32, device=device)
                self.off = torch.zeros(n_blocks + 1, dtype=torch.int64, device=device)
                if not self.raw.is_cuda:
                    raise RuntimeError("StreamWindow needs CUDA device memory")
                torch.cuda.synchronize()
                handles = [[reduce_tensor(getattr(self, k)) for k in names]]
            except Exception as e:                               # noqa: BLE001 -- reported to every rank below
                handles = [("error", f"{type(e).__name__}: {e}"[:300])]
        dist.broadcast_object_list(handles, src=root)
        if isinstance(handles[0], tuple) and handles[0][0] == "error":
            err = handles[0][1]
        elif rank != root:
            try:
                for k, (fn, a) in zip(names, handles[0]):
                    setattr(self, k, fn(*a))                     # a view of the root's memory (device = the root's index)
                self.copy_in = torch.cuda.Stream(device=device)
                self.copy_out = torch.cuda.Stream(device=device)
            except Exception as e:                               # noqa: BLE001
                err = f"rank {rank}: {type(e).__name__}: {e}"[:300]
        errs = [None] * world
        dist.all_gather_object(errs, err)
        errs = [e for e in errs if e]
        if errs:
            for k in names:
                setattr(self, k, None)
            raise RuntimeError("StreamWindow could not be set up: " + errs[0])

    def close(self):
        """Collective: the peers unmap the window, then the root lets go of it."""
        import torch
        import torch.distributed as dist
        if self.rank != self.root:
            for k in ("raw", "packed", "lens", "off"):
                setattr(self, k, None)
        torch.cuda.synchronize()
        dist.barrier()
        torch.cuda.ipc_collect()
        if self.rank == self.root:
            for k in ("raw", "packed", "lens", "off"):
                setattr(self, k, None)

    def ranges(self, pieces: int):
        """This rank's block range cut into at most `pieces` sub-ranges."""
        a, b = strong_range(self.rank, self.world, self.n_blocks)
        k = max(1, min(pieces, b - a))
        return [(a + (b - a) * p // k, a + (b - a) * (p + 1) // k) for p in range(k)] if b > a else []


def _peer_copy(dst, src, stream):
    """dst <- src between two GPUs, ordered on `stream` of this rank's device (a copy-engine transfer).  Not Tensor.copy_:
    that one runs on the SOURCE device's current stream with an event hand-shake either side, which (measured) lets the
    first kernel start only after the last queued pull."""
    assert dst.is_contiguous() and src.is_contiguous() and dst.numel() * dst.element_size() == src.numel() * src.element_size()
    from . import native
    native.check(native.lib().lz4b200_peer_copy(dst.data_ptr(), src.data_ptr(), dst.numel() * dst.element_size(), stream.cuda_stream),
                 "lz4b200_peer_copy")


def _mark(trace, what, stream=None):
    if trace is not None:
        import torch
        ev = torch.cuda.Event(enable_timing=True)
        ev.record(stream if stream is not None else torch.cuda.current_stream())
        trace.append((what, ev))


def _pull(win_slice, stream, trace=None):
    """Window -> a new local buffer, on `stream`; returns (buffer, event)."""
    import torch
    buf = torch.empty(win_slice.numel(), dtype=win_slice.dtype, device=stream.device)
    stream.wait_stream(torch.cuda.current_stream())              # (the buffer's previous life on the current stream is over)
    _peer_copy(buf, win_slice, stream)
    ev = torch.cuda.Event()
    ev.record(stream)
    buf.record_stream(stream)
    _mark(trace, "pulled", stream)
    return buf, ev


def _push(win_slice, local, stream, trace=None):
    """A local buffer -> the window, on `stream`, after everything queued so far on the current stream."""
    import torch
    stream.wait_stream(torch.cuda.current_stream())
    _peer_copy(win_slice, local, stream)
    local.record_stream(stream)
    _mark(trace, "pushed", stream)


def _halves(f):
    """(launch, finish) of a codec function: its own two halves when it has them, else the whole call up front."""
    if hasattr(f, "launch"):
        return f.launch, f.finish
    return (lambda *a, **k: f(*a, **k)), (lambda h: h)


def encode_stream_window(win: "StreamWindow", encode_local, pieces: int = 4, trace=None):
    """The raw stream is in win.raw on the root (complete before the call).  On return (all ranks) win.lens, win.off and
    win.packed[:win.off[-1]] hold the encoded stream in stream order; the root gets (lens, off, packed) views.
    A peer queues ALL its pulls and, behind each one's event, that piece's kernels, without touching the host in
    between (a host read-back mid-way would queue behind the bulk transfers on the copy engines)."""
    import torch
    import torch.distributed as dist
    bs, rank, root = win.block_size, win.rank, win.root
    launch, finish = _halves(encode_local)
    torch.cuda.synchronize()
    dist.barrier()                                               # the root's raw bytes are in place
    _mark(trace, "start")
    rng = win.ranges(pieces)
    hs = []
    if rank == root:
        for lo, hi in rng:
            hs.append(launch(win.raw[lo * bs: hi * bs], hi - lo)); _mark(trace, "encoded")
    else:
        pulls = [_pull(win.raw[lo * bs: hi * bs], win.copy_in, trace) for lo, hi in rng]    # all queued: they run back to back
        for (lo, hi), (buf, ev) in zip(rng, pulls):
            torch.cuda.current_stream().wait_event(ev)
            hs.append(launch(buf, hi - lo)); _mark(trace, "encoded")
    torch.cuda.current_stream().synchronize()
    parts = [finish(h) for h in hs]
    total = sum(int(pk.numel()) for pk, _ in parts)
    totals = _all_gather_i64(total, win.device)
    pos = sum(totals[:rank])
    for (lo, hi), (pk, ln) in zip(rng, parts):                   # own payloads and lengths into the window, in stream order
        if rank == root:
            win.packed[pos: pos + pk.numel()] = pk
            win.lens[lo:hi] = ln
        else:
            _push(win.packed[pos: pos + pk.numel()], pk, win.copy_out, trace)
            _push(win.lens[lo:hi], ln, win.copy_out)
        pos += int(pk.numel())
    torch.cuda.synchronize()
    _mark(trace, "landed")
    dist.barrier()                                               # everybody's bytes have landed
    if rank != root:
        return None, None, None
    win.off[1:] = torch.cumsum(win.lens.to(torch.int64), 0)
    return win.lens, win.off, win.packed[: sum(totals)]


def decode_stream_window(win: "StreamWindow", decode_local, pieces: int = 4, trace=None):
    """win.lens / win.off / win.packed hold an encoded stream on the root (as encode_stream_window leaves them); on return
    win.raw holds the decoded stream (returned on the root).  A peer pulls piece p+1 and pushes piece p-1 while piece p
    is in the kernel; everything is queued up front."""
    import torch
    import torch.distributed as dist
    bs, rank, root = win.block_size, win.rank, win.root
    launch, finish = _halves(decode_local)
    torch.cuda.synchronize()
    dist.barrier()
    rng = win.ranges(pieces)
    _mark(trace, "start")
    hs = []
    if rank == root and rng:
        a, b = rng[0][0], rng[-1][1]
        edge = win.off[torch.tensor([lo for lo, _ in rng] + [b], device=win.off.device)].tolist()
        for i, (lo, hi) in enumerate(rng):
            hs.append(launch(win.packed[edge[i]: edge[i + 1]], win.lens[lo:hi], hi - lo, out=win.raw[lo * bs: hi * bs]))
            _mark(trace, "decoded")
    elif rng:
        a, b = rng[0][0], rng[-1][1]
        off, _ = _pull(win.off[a: b + 1], win.copy_in)           # 8 bytes per block: where my payloads are
        lens, ev = _pull(win.lens[a:b], win.copy_in)
        ev.synchronize()
        edge = off[torch.tensor([lo - a for lo, _ in rng] + [b - a], device=off.device)].tolist()
        pulls = [_pull(win.packed[edge[i]: edge[i + 1]], win.copy_in, trace) for i in range(len(rng))]
        for i, (lo, hi) in enumerate(rng):
            torch.cuda.current_stream().wait_event(pulls[i][1])
            h = launch(pulls[i][0], lens[lo - a: hi - a], hi - lo)
            _mark(trace, "decoded")
            raw = h[0] if isinstance(h, tuple) else h
            _push(win.raw[lo * bs: hi * bs], raw, win.copy_out, trace)
            hs.append(h)
    torch.cuda.synchronize()
    for h in hs:
        finish(h)
    dist.barrier()
    return win.raw if rank == root else None


def gpu_codec(ctx, block_size: int, hc: bool = False):
    """(encode_local, decode_local) on device tensors through the C ABI (lz4b200_encode_batch / compact / decode_batch).
    Each also comes in two halves -- f.launch(...) queues the kernels on the current stream without touching the host,
    f.finish(handle) is called after the stream has been synchronized -- so a caller can queue several pieces behind
    their transfers and pay for one synchronization."""
    import torch
    from . import batch

    def encode_launch(raw, m):
        slot = block_size + block_size // 255 + 16
        so, do, sl, dc = batch.uniform_layout(m, block_size, slot, raw.device)
        slots = torch.empty(m * slot, dtype=torch.uint8, device=raw.device)
        lens = torch.zeros(m, dtype=torch.int32, device=raw.device)
        batch.encode(ctx, raw, so, sl, slots, do, dc, lens, hc=hc)
        off = torch.zeros(m + 1, dtype=torch.int64, device=raw.device)
        packed = torch.empty(m * slot, dtype=torch.uint8, device=raw.device)
        batch.compact(ctx, slots, do, lens, packed, off)
        return packed, lens, off, (lens <= 0).sum()

    def encode_finish(h):
        packed, lens, off, bad = h
        assert int(bad) == 0, "encode failed"
        return packed[: int(off[-1].item())], lens

    def encode_local(raw, m):
        h = encode_launch(raw, m)
        torch.cuda.current_stream().synchronize()               # (this stream only)
        return encode_finish(h)

    def decode_launch(packed, lens, m, out=None):
        off = torch.zeros(m + 1, dtype=torch.int64, device=packed.device)
        off[1:] = torch.cumsum(lens.to(torch.int64), 0)
        so, _, sl, _ = batch.uniform_layout(m, block_size, block_size, packed.device)
        if out is None:
            out = torch.empty(m * block_size, dtype=torch.uint8, device=packed.device)
        used = torch.zeros(m, dtype=torch.int32, device=packed.device)
        batch.decode(ctx, packed, off[:-1].contiguous(), lens, out, so, sl, used, known=True)
        return out, (used != lens).sum()

    def decode_finish(h):
        out, bad = h
        assert int(bad) == 0, "decode rejected a stream"
        return out

    def decode_local(packed, lens, m, out=None):
        h = decode_launch(packed, lens, m, out)
        torch.cuda.current_stream().synchronize()
        return decode_finish(h)

    encode_local.launch, encode_local.finish = encode_launch, encode_finish
    decode_local.launch, decode_local.finish = decode_launch, decode_finish
    return encode_local, decode_local
