"""Device-memory batches: torch owns the HBM buffers, the work is done by liblz4b200.so on raw pointers.

A batch is the GPU-native unit of work of this codec (the reference handles one block per call; LZ4Stream dispatches
one block at a time, src/LZ4/LZ4Stream.cs:239-269).  Layouts:

* raw blocks      uint8[n_blocks * block_size], block i at i * block_size
* encoder slots   uint8[n_blocks * slot], slot = MaximumOutputLength(block_size) (or block_size for LZ4Stream/Wrap caps)
* packed payload  uint8[sum(len)], block i at off[i] (exclusive prefix sum, int64[n_blocks + 1])
"""
from __future__ import annotations

import torch

from . import native
from .codec import Context


def _p(t: torch.Tensor) -> int:
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


def compact(ctx: Context, slots: torch.Tensor, slot_off, lens, packed, out_off):
    """out_off: int64[n+1]; packed may be None to compute only the offsets."""
    native.check(native.lib().lz4b200_compact(ctx.handle, _p(slots), _p(slot_off), _p(lens),
                                              _p(packed) if packed is not None else 0, _p(out_off), lens.numel(), _stream()),
                 "compact")
