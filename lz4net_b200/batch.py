"""Device-memory batches: torch owns the HBM buffers, the work is done by liblz4b200.so on raw pointers.

A batch is the GPU-native unit of work of this codec (the reference handles one block per call; LZ4Stream dispatches
one block at a time, src/LZ4/LZ4Stream.cs:239-269).  Layouts:

* raw blocks      uint8[n_blocks * block_size], block i at i * block_size
* encoder slots   uint8[n_blocks * slot], slot = MaximumOutputLength(block_size) (or block_size for LZ4Stream/Wrap caps)
* packed payload  uint8[sum(len)], block i at off[i] (exclusive prefix sum, int64[n_blocks + 1])

The mixed-memory helpers (encode_to_host, encode_to_host_packed, decode_from_host, decode_from_host_packed) take the device side as a torch CUDA
tensor and the host side -- data, offsets, lengths, results -- as numpy arrays.  They are synchronous, ordered behind the
work already queued on the current torch stream, and move only compressed bytes over PCIe.  stream_encode_to_host and
stream_decode_to_device do the same for the LZ4Stream format: a device tensor's bytes as a stream in host memory, and back.
wrap_to_host, wrap_to_host_packed, unwrap_to_device and unwrap_to_device_packed do it for Wrap packets: inputs in a device
tensor, packets in a host array, and back.

The asynchronous helpers (synth_fill, encode, decode, measure, decode_packed, compact, wrap, wrap_packed, unwrap,
unwrap_packed) can be captured in a CUDA graph: reserve the scratch of the largest batch first, then capture, then replay
with new contents in the same tensors:

    ctx.reserve(n_blocks, hc=True)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        batch.encode(ctx, raw, src_off, src_len, slots, dst_off, dst_cap, out_len, hc=True)
        batch.compact(ctx, slots, dst_off, out_len, packed, out_off)
    g.replay()

A call whose scratch was not reserved raises Lz4B200Error (E_ARG) and leaves the capture valid.  The synchronous helpers
refuse a capturing stream the same way.

encode_to_host_packed_async and decode_from_host_async move blocks between a device tensor and a page-locked CPU tensor
without blocking the calling thread: they enqueue their work on a stream and return, so a thread that launches a model's
kernels can offload to host RAM, or prefetch back, and keep launching.  decode_from_host_packed_async,
wrap_to_host_packed_async, unwrap_to_device_async and unwrap_to_device_packed_async do the same for the packed decode and
for Wrap packets, which carry their own sizes and never exceed input + 8 bytes.  decode_from_host_at_async and
unwrap_to_device_at_async bring such an offload back from the out_off the device wrote, with no synchronisation in
between.  stream_encode_to_host_async and
stream_decode_to_device_async do it for an LZ4Stream: one byte string, one pointer and one length, that any LZ4Stream reads;
stream_decode_to_device_at_async brings such a stream back from the size the device wrote, with no synchronisation in
between.  They refuse a capturing stream.
"""
from __future__ import annotations

import numpy as np
import torch

from . import native
from .codec import Context


def _p(t: torch.Tensor) -> int:
    return t.data_ptr()


def _h(a: np.ndarray, dtype, n: int = 0) -> int:
    """Address of a host array that the library reads or writes in place: C-contiguous, of this dtype, >= n items."""
    if not (isinstance(a, np.ndarray) and a.dtype == dtype and a.flags.c_contiguous and a.size >= n):
        raise TypeError(f"expected a C-contiguous numpy {np.dtype(dtype).name} array of at least {n} items")
    return a.ctypes.data


def _d(t: torch.Tensor) -> int:
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise TypeError("expected a torch CUDA tensor")
    return t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def uniform_layout(n_blocks: int, block_size: int, slot: int, device):
    idx = torch.arange(n_blocks, dtype=torch.int64, device=device)
    return idx * block_size, idx * slot, torch.full((n_blocks,), block_size, dtype=torch.int32, device=device), \
        torch.full((n_blocks,), slot, dtype=torch.int32, device=device)


def synth_fill(ctx: Context, dst: torch.Tensor, n_blocks: int, block_size: int, cls: int, seed: int = 1, first_block: int = 0):
    native.check(native.lib().lz4b200_synth_fill(ctx.handle, _p(dst), n_blocks, block_size, cls, seed, first_block, _stream()),
                 "synth_fill")


def encode(ctx: Context, raw: torch.Tensor, src_off, src_len, slots: torch.Tensor, dst_off, dst_cap, out_len, hc: bool = False):
    """Asynchronous on the current torch stream."""
    ctx.encode_batch_ptr(_p(raw), _p(src_off), _p(src_len), _p(slots), _p(dst_off), _p(dst_cap), _p(out_len),
                         src_off.numel(), hc=hc, device=True, stream=_stream())


def decode(ctx: Context, comp: torch.Tensor, src_off, src_len, out: torch.Tensor, dst_off, dst_cap, out_len, known: bool = True):
    ctx.decode_batch_ptr(_p(comp), _p(src_off), _p(src_len), _p(out), _p(dst_off), _p(dst_cap), _p(out_len),
                         src_off.numel(), known=known, device=True, stream=_stream())


def measure(ctx: Context, comp: torch.Tensor, src_off, src_len, out_len, dst_cap=None, known: bool = False):
    """out_len[i] = what decode(..., dst_cap, out_len, known) would store, without decoding; dst_cap=None (unknown size only)
    = no limit.  Asynchronous on the current torch stream."""
    ctx.measure_batch_ptr(_p(comp), _p(src_off), _p(src_len), _p(dst_cap) if dst_cap is not None else None, _p(out_len),
                          src_off.numel(), known=known, device=True, stream=_stream())


def decode_packed(ctx: Context, comp: torch.Tensor, src_off, src_len, out: torch.Tensor, out_off, out_len):
    """Unknown-size decode into packed output (lz4b200_decode_batch_packed): block i lands at out + out_off[i] (int64[n+1],
    out_off[n] = the total) when the total fits out.numel() bytes; otherwise out is untouched and out_len holds the sizes.
    Asynchronous on the current torch stream: read out_off[n] after a synchronise to learn which happened."""
    native.check(native.lib().lz4b200_decode_batch_packed(ctx.handle, _p(comp), _p(src_off), _p(src_len), _p(out), out.numel(),
                                                          _p(out_off), _p(out_len), src_off.numel(), _stream()),
                 "decode_batch_packed")


def wrap(ctx: Context, raw: torch.Tensor, src_off, src_len, packets: torch.Tensor, dst_off, dst_cap, out_len, hc: bool = False):
    """LZ4Codec.Wrap / WrapHC packets in device memory (lz4b200_wrap_batch_device): packet i of input i lands at
    packets + dst_off[i] (dst_cap[i] >= src_len[i] + 8); out_len[i] = its size or LZ4B200_E_ARG.  Asynchronous on the
    current torch stream."""
    native.check(native.lib().lz4b200_wrap_batch_device(ctx.handle, _p(raw), _p(src_off), _p(src_len), int(hc), _p(packets),
                                                        _p(dst_off), _p(dst_cap), _p(out_len), src_off.numel(), _stream()),
                 "wrap_batch_device")


def wrap_packed(ctx: Context, raw: torch.Tensor, src_off, src_len, slots: torch.Tensor, slot_off, slot_cap, out_len,
                packed: torch.Tensor, out_off, hc: bool = False):
    """wrap() into the slots, then compact(): the packets back to back at packed + out_off[i] (int64[n+1], out_off[n] =
    the total).  A packet with a negative out_len occupies no bytes.  Asynchronous on the current torch stream."""
    wrap(ctx, raw, src_off, src_len, slots, slot_off, slot_cap, out_len, hc=hc)
    compact(ctx, slots, slot_off, out_len, packed, out_off)


def unwrap(ctx: Context, packets: torch.Tensor, src_off, src_len, out: torch.Tensor, dst_off, dst_cap, out_len):
    """Mirror image of wrap() (lz4b200_unwrap_batch_device): out_len[i] = bytes restored, LZ4B200_E_FORMAT or E_ARG.
    Asynchronous on the current torch stream."""
    native.check(native.lib().lz4b200_unwrap_batch_device(ctx.handle, _p(packets), _p(src_off), _p(src_len), _p(out),
                                                          _p(dst_off), _p(dst_cap), _p(out_len), src_off.numel(), _stream()),
                 "unwrap_batch_device")


def unwrap_packed(ctx: Context, packets: torch.Tensor, src_off, src_len, out: torch.Tensor, out_off, out_len):
    """Unwrap into packed output sized from the headers (lz4b200_unwrap_batch_packed), in the shape of decode_packed:
    packet i lands at out + out_off[i] when out_off[n] fits out.numel() bytes; otherwise out is untouched and out_len
    holds the sizes.  Asynchronous on the current torch stream."""
    native.check(native.lib().lz4b200_unwrap_batch_packed(ctx.handle, _p(packets), _p(src_off), _p(src_len), _p(out), out.numel(),
                                                          _p(out_off), _p(out_len), src_off.numel(), _stream()),
                 "unwrap_batch_packed")


def encode_to_host(ctx: Context, raw: torch.Tensor, src_off, src_len, dst: np.ndarray, dst_off, dst_cap, out_len, hc: bool = False):
    """Blocks of a device tensor encoded into slots of a host array (lz4b200_encode_batch, MEM_DEVICE_TO_HOST): block i
    reads raw + src_off[i] and its compressed bytes land at dst + dst_off[i] (only the out_len[i] bytes it produced).
    src_off / dst_off int64, src_len / dst_cap / out_len int32 numpy arrays."""
    n = len(src_off)
    ctx.encode_batch_ptr(_d(raw), _h(src_off, np.int64), _h(src_len, np.int32, n), _h(dst, np.uint8), _h(dst_off, np.int64, n),
                         _h(dst_cap, np.int32, n), _h(out_len, np.int32, n), n, hc=hc, stream=_stream(),
                         mem=native.MEM_DEVICE_TO_HOST)


def encode_to_host_packed(ctx: Context, raw: torch.Tensor, src_off, src_len, dst_cap, dst: np.ndarray, out_off, out_len,
                          hc: bool = False) -> int:
    """The same, packed (lz4b200_encode_batch_packed_from_device): block i's bytes land at dst + out_off[i], back to back in
    block order, out_off (int64[n+1]) [n] = the total, which is returned.  Raises when the total exceeds dst.nbytes."""
    n = len(src_off)
    native.check(native.lib().lz4b200_encode_batch_packed_from_device(
        ctx.handle, _d(raw), _h(src_off, np.int64), _h(src_len, np.int32, n), _h(dst_cap, np.int32, n), _h(dst, np.uint8),
        dst.nbytes, _h(out_off, np.int64, n + 1), _h(out_len, np.int32, n), n,
        native.MODE_HC if hc else native.MODE_FAST, _stream()), "encode_batch_packed_from_device")
    return int(out_off[n])


def decode_from_host(ctx: Context, comp: np.ndarray, src_off, src_len, out: torch.Tensor, dst_off, dst_cap, out_len,
                     known: bool = True):
    """Compressed blocks in a host array decoded into a device tensor (lz4b200_decode_batch, MEM_HOST_TO_DEVICE): block i
    reads comp + src_off[i] and is decoded in place at out + dst_off[i], nothing written outside its dst_cap[i] bytes."""
    n = len(src_off)
    ctx.decode_batch_ptr(_h(comp, np.uint8), _h(src_off, np.int64), _h(src_len, np.int32, n), _d(out), _h(dst_off, np.int64, n),
                         _h(dst_cap, np.int32, n), _h(out_len, np.int32, n), n, known=known, stream=_stream(),
                         mem=native.MEM_HOST_TO_DEVICE)


def decode_from_host_packed(ctx: Context, comp: np.ndarray, src_off, src_len, out: torch.Tensor, out_off, out_len) -> int:
    """Compressed blocks in a host array whose decoded sizes nobody stored, decoded into a device tensor, packed
    (lz4b200_decode_batch_packed_to_device): block i lands at out + out_off[i] (int64[n+1], out_off[n] = the total, which is
    returned) when the total fits out.nbytes.  Otherwise nothing is written outside `out`, its bytes are unspecified, and
    out_len holds the sizes (negative for malformed blocks): allocate the returned total and call again.  The compressed
    bytes cross PCIe once."""
    n = len(src_off)
    off, res = _h(out_off, np.int64, n + 1), _h(out_len, np.int32, n)
    native.check(native.lib().lz4b200_decode_batch_packed_to_device(
        ctx.handle, _h(comp, np.uint8), _h(src_off, np.int64), _h(src_len, np.int32, n), _d(out), out.nbytes, off, res, n,
        _stream()), "decode_batch_packed_to_device")
    return int(out_off[n])


def _pinned(t: torch.Tensor, dtype, n: int, what: str, device_ok: bool = False) -> int:
    """Address of a contiguous tensor of this dtype and at least n items that the device reaches after the call has
    returned: page-locked CPU memory, or with device_ok a CUDA tensor.  An empty tensor where none is needed is not read."""
    if n == 0 and isinstance(t, torch.Tensor) and t.numel() == 0:
        return t.data_ptr()
    if not (isinstance(t, torch.Tensor) and t.dtype == dtype and t.is_contiguous() and t.numel() >= n):
        raise TypeError(f"{what}: expected a contiguous torch {dtype} tensor of at least {n} items")
    if not ((device_ok and t.is_cuda) or (t.device.type == "cpu" and t.is_pinned())):
        raise TypeError(f"{what}: expected a page-locked CPU tensor (pin_memory())" + (" or a CUDA tensor" if device_ok else ""))
    return t.data_ptr()


def _stream_of(stream) -> int:
    return stream.cuda_stream if stream is not None else _stream()


def encode_to_host_packed_async(ctx: Context, raw: torch.Tensor, src_off, src_len, dst_cap, dst: torch.Tensor, out_off: torch.Tensor,
                                out_len: torch.Tensor, hc: bool = False, stream=None):
    """encode_to_host_packed without blocking (lz4b200_encode_batch_packed_from_device_async): block i of raw + src_off[i] is
    encoded and its bytes land at dst + out_off[i], back to back, out_off[n] = the total.  dst is a page-locked CPU uint8
    tensor; out_off (int64[n+1]) and out_len (int32[n]) are CUDA or page-locked CPU tensors, written by the device;
    src_off / src_len / dst_cap are numpy arrays, read during the call.  Enqueued on `stream` (default: the current torch
    stream) behind the work already there; returns at once.  The caller keeps raw, dst, out_off and out_len alive and
    untouched until the stream has passed the call.  When the total exceeds dst.numel() the call still succeeds: out_off and
    out_len are filled and the bytes of dst are unspecified; check out_off[n] after synchronising."""
    n = len(src_off)
    d, off, res = (_pinned(dst, torch.uint8, 0, "dst"), _pinned(out_off, torch.int64, n + 1, "out_off", True),
                   _pinned(out_len, torch.int32, n, "out_len", True))
    native.check(native.lib().lz4b200_encode_batch_packed_from_device_async(
        ctx.handle, _d(raw), _h(src_off, np.int64), _h(src_len, np.int32, n), _h(dst_cap, np.int32, n), d, dst.numel(), off, res,
        n, native.MODE_HC if hc else native.MODE_FAST, _stream_of(stream)), "encode_batch_packed_from_device_async")


def decode_from_host_async(ctx: Context, comp: torch.Tensor, src_off, src_len, out: torch.Tensor, dst_off, dst_cap,
                           out_len: torch.Tensor, known: bool = True, stream=None):
    """decode_from_host without blocking (lz4b200_decode_batch_to_device_async): block i of comp + src_off[i] is decoded in
    place at out + dst_off[i], nothing written outside its dst_cap[i] bytes.  comp is a page-locked CPU uint8 tensor;
    out_len (int32[n]) a CUDA or page-locked CPU tensor, written by the device; src_off / src_len / dst_off / dst_cap are
    numpy arrays, read during the call.  Enqueued on `stream` (default: the current torch stream) behind the work already
    there; returns at once.  The caller keeps comp, out and out_len alive and untouched until the stream has passed the
    call."""
    n = len(src_off)
    c, res = _pinned(comp, torch.uint8, 0, "comp"), _pinned(out_len, torch.int32, n, "out_len", True)
    native.check(native.lib().lz4b200_decode_batch_to_device_async(
        ctx.handle, c, _h(src_off, np.int64), _h(src_len, np.int32, n), _d(out), _h(dst_off, np.int64, n), _h(dst_cap, np.int32, n),
        res, n, int(known), _stream_of(stream)), "decode_batch_to_device_async")


def decode_from_host_packed_async(ctx: Context, comp: torch.Tensor, src_off, src_len, out: torch.Tensor, out_off: torch.Tensor,
                                  out_len: torch.Tensor, stream=None):
    """decode_from_host_packed without blocking (lz4b200_decode_batch_packed_to_device_async): blocks whose decoded sizes
    nobody stored, decoded into `out` back to back, block i at out_off[i], out_off[n] = the total.  comp is a page-locked CPU
    uint8 tensor; out_off (int64[n+1]) and out_len (int32[n]) are CUDA or page-locked CPU tensors, written by the device;
    src_off / src_len are numpy arrays, read during the call.  Enqueued on `stream` (default: the current torch stream);
    returns at once.  When the total exceeds out.nbytes the call still succeeds: nothing is written outside `out`, its
    bytes are unspecified, and out_len holds the sizes; check out_off[n] after synchronising."""
    n = len(src_off)
    c = _pinned(comp, torch.uint8, 0, "comp")
    off, res = _pinned(out_off, torch.int64, n + 1, "out_off", True), _pinned(out_len, torch.int32, n, "out_len", True)
    native.check(native.lib().lz4b200_decode_batch_packed_to_device_async(
        ctx.handle, c, _h(src_off, np.int64), _h(src_len, np.int32, n), _d(out), out.nbytes, off, res, n, _stream_of(stream)),
        "decode_batch_packed_to_device_async")


def wrap_to_host_packed_async(ctx: Context, raw: torch.Tensor, src_off, src_len, dst: torch.Tensor, out_off: torch.Tensor,
                              out_len: torch.Tensor, hc: bool = False, stream=None):
    """wrap_to_host_packed without blocking (lz4b200_wrap_batch_packed_from_device_async): the Wrap / WrapHC packet of
    raw + src_off[i] lands at dst + out_off[i], back to back, out_off[n] = the total; sum(src_len + 8) bytes of dst are
    always enough.  dst is a page-locked CPU uint8 tensor; out_off (int64[n+1]) and out_len (int32[n]) are CUDA or
    page-locked CPU tensors, written by the device; src_off / src_len are numpy arrays, read during the call.  Enqueued on
    `stream` (default: the current torch stream); returns at once.  When the total exceeds dst.numel() the call still
    succeeds: out_off and out_len are filled and nothing is written outside dst; check out_off[n] after synchronising."""
    n = len(src_off)
    d, off, res = (_pinned(dst, torch.uint8, 0, "dst"), _pinned(out_off, torch.int64, n + 1, "out_off", True),
                   _pinned(out_len, torch.int32, n, "out_len", True))
    native.check(native.lib().lz4b200_wrap_batch_packed_from_device_async(
        ctx.handle, _d(raw), _h(src_off, np.int64), _h(src_len, np.int32, n), int(hc), d, dst.numel(), off, res, n,
        _stream_of(stream)), "wrap_batch_packed_from_device_async")


def unwrap_to_device_async(ctx: Context, packets: torch.Tensor, src_off, src_len, out: torch.Tensor, dst_off, dst_cap,
                           out_len: torch.Tensor, stream=None):
    """unwrap_to_device without blocking (lz4b200_unwrap_batch_to_device_async): packet i of packets + src_off[i] is
    restored at out + dst_off[i], nothing written outside its dst_cap[i] bytes; out_len[i] = bytes restored,
    LZ4B200_E_FORMAT or E_ARG.  The headers are read on the device, so the packets may still be being written by work
    queued on the stream before the call.  packets is a page-locked CPU uint8 tensor; out_len (int32[n]) a CUDA or
    page-locked CPU tensor; src_off / src_len / dst_off / dst_cap are numpy arrays, read during the call."""
    n = len(src_off)
    p, res = _pinned(packets, torch.uint8, 0, "packets"), _pinned(out_len, torch.int32, n, "out_len", True)
    native.check(native.lib().lz4b200_unwrap_batch_to_device_async(
        ctx.handle, p, _h(src_off, np.int64), _h(src_len, np.int32, n), _d(out), _h(dst_off, np.int64, n), _h(dst_cap, np.int32, n),
        res, n, _stream_of(stream)), "unwrap_batch_to_device_async")


def unwrap_to_device_packed_async(ctx: Context, packets: torch.Tensor, src_off, src_len, out: torch.Tensor, out_off: torch.Tensor,
                                  out_len: torch.Tensor, stream=None):
    """unwrap_to_device_packed without blocking (lz4b200_unwrap_batch_packed_to_device_async): packet i lands at
    out + out_off[i] (int64[n+1], written by the device, out_off[n] = the total) when the total fits out.nbytes.  Otherwise
    the call still succeeds: nothing is written outside `out`, its bytes are unspecified, and out_len[i] is non-negative
    exactly for the well-formed packets, where it is the size.  The headers are read on the device."""
    n = len(src_off)
    p = _pinned(packets, torch.uint8, 0, "packets")
    off, res = _pinned(out_off, torch.int64, n + 1, "out_off", True), _pinned(out_len, torch.int32, n, "out_len", True)
    native.check(native.lib().lz4b200_unwrap_batch_packed_to_device_async(
        ctx.handle, p, _h(src_off, np.int64), _h(src_len, np.int32, n), _d(out), out.nbytes, off, res, n, _stream_of(stream)),
        "unwrap_batch_packed_to_device_async")


def _at_args(comp, src_cap, src_off, out_len, n, what):
    """The page-locked source, its readable bytes and the device-read offsets of the *_at_async calls."""
    c = _pinned(comp, torch.uint8, 0, what)
    if not 0 <= src_cap <= comp.numel():
        raise ValueError(f"src_cap: {src_cap} is not within the {comp.numel()} bytes of {what}")
    return c, _pinned(src_off, torch.int64, n + 1, "src_off", True), _pinned(out_len, torch.int32, n, "out_len", True)


def decode_from_host_at_async(ctx: Context, comp: torch.Tensor, src_cap: int, src_off: torch.Tensor, out: torch.Tensor, dst_off,
                              dst_cap, out_len: torch.Tensor, known: bool = True, stream=None):
    """decode_from_host_async whose block offsets are read on the device, when the call's work runs
    (lz4b200_decode_batch_to_device_at_async): block i spans comp[src_off[i]:src_off[i+1]] and is decoded at
    out + dst_off[i].  src_off (int64[n+1]) is a CUDA or page-locked CPU tensor -- the out_off an
    encode_to_host_packed_async has just written, for one -- so the round trip needs no synchronisation in between.  Only
    the first src_cap bytes of comp are read.  A span that is not within them, runs backwards or is longer than
    compress_bound(dst_cap[i]) gets out_len[i] = LZ4B200_E_ARG and nothing written; so does every block when
    src_off[n] > src_cap.  dst_off / dst_cap are numpy arrays, read during the call."""
    n = len(dst_off)
    c, off, res = _at_args(comp, src_cap, src_off, out_len, n, "comp")
    native.check(native.lib().lz4b200_decode_batch_to_device_at_async(
        ctx.handle, c, src_cap, off, _d(out), _h(dst_off, np.int64), _h(dst_cap, np.int32, n), res, n, int(known),
        _stream_of(stream)), "decode_batch_to_device_at_async")


def unwrap_to_device_at_async(ctx: Context, packets: torch.Tensor, src_cap: int, src_off: torch.Tensor, out: torch.Tensor, dst_off,
                              dst_cap, out_len: torch.Tensor, stream=None):
    """unwrap_to_device_async whose packet offsets are read on the device (lz4b200_unwrap_batch_to_device_at_async): the
    out_off a wrap_to_host_packed_async has just written can be passed as src_off.  A packet span above dst_cap[i] + 8
    bytes is LZ4B200_E_ARG; otherwise as decode_from_host_at_async."""
    n = len(dst_off)
    p, off, res = _at_args(packets, src_cap, src_off, out_len, n, "packets")
    native.check(native.lib().lz4b200_unwrap_batch_to_device_at_async(
        ctx.handle, p, src_cap, off, _d(out), _h(dst_off, np.int64), _h(dst_cap, np.int32, n), res, n, _stream_of(stream)),
        "unwrap_batch_to_device_at_async")


def stream_encode_to_host_async(ctx: Context, raw: torch.Tensor, dst: torch.Tensor, out_size: torch.Tensor,
                                block_size: int = 1 << 20, hc: bool = False, stream=None):
    """stream_encode_to_host without blocking (lz4b200_stream_encode_from_device_async): the LZ4Stream of raw's bytes, cut
    into block_size chunks, is written at the start of dst, and its size to out_size[0].  dst is a page-locked CPU uint8
    tensor of at least lz4b200_stream_bound bytes; out_size (int64[1]) a CUDA or page-locked CPU tensor, written by the
    device.  Enqueued on `stream` (default: the current torch stream) behind the work already there; returns at once.  The
    caller keeps raw, dst and out_size alive and untouched until the stream has passed the call."""
    d, size = _pinned(dst, torch.uint8, 0, "dst"), _pinned(out_size, torch.int64, 1, "out_size", True)
    r = _flat_bytes(raw)
    native.check(native.lib().lz4b200_stream_encode_from_device_async(
        ctx.handle, r.data_ptr(), r.numel(), block_size, int(hc), d, dst.numel(), size, _stream_of(stream)),
        "stream_encode_from_device_async")


def stream_decode_to_device_async(ctx: Context, wire: torch.Tensor, n: int, out: torch.Tensor, out_size: torch.Tensor,
                                  stream=None):
    """stream_decode_to_device without blocking (lz4b200_stream_decode_to_device_async): the LZ4Stream in the first n
    bytes of wire is decoded into out's bytes, from its first byte.  wire is a page-locked CPU uint8 tensor that holds the
    whole stream when the call is made: its headers are read during the call.  out_size (int64[1]) is a CUDA or
    page-locked CPU tensor that the device sets to the decoded size, or to LZ4B200_E_FORMAT when a chunk does not decode.
    A malformed header or an `out` too small raises Lz4B200Error (E_FORMAT, E_ARG) with nothing enqueued.  Enqueued on
    `stream` (default: the current torch stream); returns at once.  The caller keeps wire, out and out_size alive and
    untouched until the stream has passed the call."""
    w, size = _pinned(wire, torch.uint8, n, "wire"), _pinned(out_size, torch.int64, 1, "out_size", True)
    o = _flat_bytes(out)
    native.check(native.lib().lz4b200_stream_decode_to_device_async(
        ctx.handle, w, n, o.data_ptr(), o.numel(), size, _stream_of(stream)), "stream_decode_to_device_async")


def stream_decode_to_device_at_async(ctx: Context, wire: torch.Tensor, src_cap: int, src_size: torch.Tensor, out: torch.Tensor,
                                     out_size: torch.Tensor, block_size: int = 1 << 20, stream=None):
    """stream_decode_to_device_async whose stream size is read on the device, when the call's work runs
    (lz4b200_stream_decode_to_device_at_async): src_size (int64[1]) is a CUDA or page-locked CPU tensor -- the out_size a
    stream_encode_to_host_async has just written, for one -- so the round trip needs no synchronisation in between.  The
    headers are walked on the device; only the first src_cap bytes of wire (page-locked) are read.  block_size is the chunk
    size the stream was written with.  out_size (int64[1], CUDA or page-locked) is set to the decoded size, or to
    LZ4B200_E_ARG (a size outside [0, src_cap], a chunk above block_size, more chunks or bytes than out holds) or
    LZ4B200_E_FORMAT (a malformed header, a chunk that does not decode)."""
    w = _pinned(wire, torch.uint8, 0, "wire")
    if not 0 <= src_cap <= wire.numel():
        raise ValueError(f"src_cap: {src_cap} is not within the {wire.numel()} bytes of wire")
    size, res = _pinned(src_size, torch.int64, 1, "src_size", True), _pinned(out_size, torch.int64, 1, "out_size", True)
    o = _flat_bytes(out)
    native.check(native.lib().lz4b200_stream_decode_to_device_at_async(
        ctx.handle, w, src_cap, size, block_size, o.data_ptr(), o.numel(), res, _stream_of(stream)),
        "stream_decode_to_device_at_async")


def wrap_to_host(ctx: Context, raw: torch.Tensor, src_off, src_len, dst: np.ndarray, dst_off, dst_cap, out_len, hc: bool = False):
    """Wrap / WrapHC packets of a device tensor's inputs written into slots of a host array (lz4b200_wrap_batch_from_device):
    packet i of raw + src_off[i] lands at dst + dst_off[i] (dst_cap[i] >= src_len[i] + 8), only its out_len[i] bytes.
    src_off / dst_off int64, src_len / dst_cap / out_len int32 numpy arrays."""
    n = len(src_off)
    native.check(native.lib().lz4b200_wrap_batch_from_device(
        ctx.handle, _d(raw), _h(src_off, np.int64), _h(src_len, np.int32, n), int(hc), _h(dst, np.uint8), _h(dst_off, np.int64, n),
        _h(dst_cap, np.int32, n), _h(out_len, np.int32, n), n, _stream()), "wrap_batch_from_device")


def wrap_to_host_packed(ctx: Context, raw: torch.Tensor, src_off, src_len, dst: np.ndarray, out_off, out_len,
                        hc: bool = False) -> int:
    """The same packets back to back in a host array (lz4b200_wrap_batch_packed_from_device): packet i at dst + out_off[i],
    out_off (int64[n+1]) [n] = the total, which is returned.  sum(src_len + 8) bytes of dst are always enough; raises when
    the packets do not fit dst.nbytes."""
    n = len(src_off)
    native.check(native.lib().lz4b200_wrap_batch_packed_from_device(
        ctx.handle, _d(raw), _h(src_off, np.int64), _h(src_len, np.int32, n), int(hc), _h(dst, np.uint8), dst.nbytes,
        _h(out_off, np.int64, n + 1), _h(out_len, np.int32, n), n, _stream()), "wrap_batch_packed_from_device")
    return int(out_off[n])


def unwrap_to_device(ctx: Context, packets: np.ndarray, src_off, src_len, out: torch.Tensor, dst_off, dst_cap, out_len):
    """Packets in a host array unwrapped into a device tensor (lz4b200_unwrap_batch_to_device): packet i of
    packets + src_off[i] is restored at out + dst_off[i], nothing written outside its dst_cap[i] bytes; out_len[i] = bytes
    restored, LZ4B200_E_FORMAT or E_ARG, as lz4b200_unwrap_batch returns."""
    n = len(src_off)
    native.check(native.lib().lz4b200_unwrap_batch_to_device(
        ctx.handle, _h(packets, np.uint8), _h(src_off, np.int64), _h(src_len, np.int32, n), _d(out), _h(dst_off, np.int64, n),
        _h(dst_cap, np.int32, n), _h(out_len, np.int32, n), n, _stream()), "unwrap_batch_to_device")


def unwrap_to_device_packed(ctx: Context, packets: np.ndarray, src_off, src_len, out: torch.Tensor, out_off, out_len) -> int:
    """Unwrap into packed output sized from the headers (lz4b200_unwrap_batch_packed_to_device): packet i lands at
    out + out_off[i] (int64[n+1]) when out_off[n] fits out.nbytes; otherwise out is untouched and out_len holds the sizes.
    Returns out_off[n]."""
    n = len(src_off)
    native.check(native.lib().lz4b200_unwrap_batch_packed_to_device(
        ctx.handle, _h(packets, np.uint8), _h(src_off, np.int64), _h(src_len, np.int32, n), _d(out), out.nbytes,
        _h(out_off, np.int64, n + 1), _h(out_len, np.int32, n), n, _stream()), "unwrap_batch_packed_to_device")
    return int(out_off[n])


def _flat_bytes(t: torch.Tensor) -> torch.Tensor:
    """The bytes of a contiguous CUDA tensor, in storage order, as a flat uint8 tensor on the same memory."""
    _d(t)
    if not t.is_contiguous():
        raise TypeError("expected a contiguous torch CUDA tensor")
    return t.reshape(-1).view(torch.uint8)


def stream_encode_to_host(ctx: Context, raw: torch.Tensor, block_size: int = 1 << 20, hc: bool = False,
                          dst: np.ndarray = None) -> np.ndarray:
    """The LZ4Stream wire bytes of a device tensor's bytes, written to host memory (lz4b200_stream_encode_from_device):
    the bytes stream_encode writes for a host copy, with only the stream bytes crossing PCIe.  `dst` (uint8, at least
    lz4b200_stream_bound bytes; pageable or page-locked) receives them, or a new array does.  Returns the view of it that
    holds the stream.  Synchronous, ordered behind the work already queued on the current torch stream."""
    r = _flat_bytes(raw)
    n = r.numel()
    cap = int(native.lib().lz4b200_stream_bound(n, block_size))
    if cap < 0:
        raise native.Lz4B200Error(f"stream_encode_to_host: bad block_size {block_size}")
    if dst is None:
        dst = np.empty(max(cap, 1), np.uint8)
    w = native.lib().lz4b200_stream_encode_from_device(ctx.handle, r.data_ptr(), n, block_size, int(hc), _h(dst, np.uint8),
                                                       dst.nbytes, _stream())
    if w < 0:
        raise native.Lz4B200Error(f"stream_encode_from_device failed with status {w}: {native.last_error()}")
    return dst[:w]


def stream_decode_to_device(ctx: Context, wire: np.ndarray, out: torch.Tensor) -> int:
    """An LZ4Stream in host memory (a uint8 numpy array) decoded into a device tensor's bytes, from its first byte
    (lz4b200_stream_decode_to_device).  Returns the decoded size; nothing is written behind it.  Raises Lz4B200Error with
    the status (E_FORMAT for a malformed stream, E_ARG when `out` is too small).  Synchronous, ordered behind the work
    already queued on the current torch stream."""
    o = _flat_bytes(out)
    r = native.lib().lz4b200_stream_decode_to_device(ctx.handle, _h(wire, np.uint8), wire.nbytes, o.data_ptr(), o.numel(),
                                                     _stream())
    if r < 0:
        raise native.Lz4B200Error(f"stream_decode_to_device failed with status {r}: {native.last_error()}")
    return int(r)


def compact(ctx: Context, slots: torch.Tensor, slot_off, lens, packed, out_off):
    """out_off: int64[n+1]; packed may be None to compute only the offsets."""
    native.check(native.lib().lz4b200_compact(ctx.handle, _p(slots), _p(slot_off), _p(lens),
                                              _p(packed) if packed is not None else 0, _p(out_off), lens.numel(), _stream()),
                 "compact")
