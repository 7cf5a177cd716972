"""Python mirror of lz4net's public surface for the accelerated path, over the C ABI.

Names, argument meaning and error behaviour follow the reference:

* ``LZ4Codec.Encode / EncodeHC / Decode / MaximumOutputLength / Wrap / WrapHC / Unwrap``  (src/LZ4/LZ4Codec.cs:313-440,510-599)
  with the C# boundary conventions: ``Encode`` of an empty input returns 0 (src/LZ4ps/LZ4Codec.cs:156-160),
  ``EncodeHC`` failure is -1 (src/LZ4ps/LZ4Codec.Safe.cs:721-723), a decode error raises (``ArgumentException`` there,
  ``ValueError`` here; src/LZ4ps/LZ4Codec.Safe.cs:539-549).
* ``CudaLZ4Service`` -- the ``ILZ4Service`` (src/LZ4/ILZ4Service.cs:30-36) implementation a maintainer would register.
* ``BlockBatch`` helpers -- the batched entry points, for torch CUDA tensors (device memory) or numpy arrays (host).

torch is used only to own device memory / streams; every call goes through ``liblz4b200.so`` with raw pointers.
"""
from __future__ import annotations

import ctypes as C
import sys
from typing import Optional

import numpy as np

from . import native

_default_ctx = None


def _offsets(lens):
    """Exclusive prefix sums (int64): where each of the items of these lengths starts when they are laid back to back."""
    return np.cumsum(lens, dtype=np.int64) - lens


def _pack(blocks):
    """Byte strings laid back to back: (uint8 buffer with 16 bytes of padding, int32 lengths, int64 offsets)."""
    lens = np.array([len(b) for b in blocks], np.int32)
    return np.frombuffer(b"".join(bytes(b) for b in blocks) + b"\0" * 16, np.uint8), lens, _offsets(lens)


class Context:
    """Owns one lz4b200_ctx (one GPU)."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        native.check(native.lib().lz4b200_create(C.byref(self._h), int(device)), "lz4b200_create")
        self.device = int(device)

    def close(self):
        if self._h:
            native.lib().lz4b200_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._h

    def set_option(self, key: str, value: int):
        native.check(native.lib().lz4b200_set_option(self._h, key.encode(), int(value)), f"set_option({key})")

    def get_option(self, key: str) -> int:
        v = native._L(0)
        native.check(native.lib().lz4b200_get_option(self._h, key.encode(), native.C.byref(v)), f"get_option({key})")
        return int(v.value)

    def synchronize(self):
        native.check(native.lib().lz4b200_synchronize(self._h), "synchronize")

    def reserve(self, max_blocks: int, hc: bool = False):
        """Grow the device scratch of device-memory calls of at most max_blocks blocks (with hc: the HC arena too), so that
        they can be captured in a CUDA graph (lz4b200_reserve)."""
        native.check(native.lib().lz4b200_reserve(self._h, int(max_blocks), int(hc)), "reserve")

    @property
    def launches(self) -> int:
        return int(native.lib().lz4b200_launch_count(self._h))

    # ---- batched calls on raw pointers -------------------------------------------------------------------------
    # mem: one of native.MEM_*; when None, device=True means MEM_DEVICE and device=False MEM_HOST
    @staticmethod
    def _mem(device, mem):
        return mem if mem is not None else native.MEM_DEVICE if device else native.MEM_HOST

    def encode_batch_ptr(self, src, src_off, src_len, dst, dst_off, dst_cap, out_len, n, hc=False, device=True, stream=0, mem=None):
        native.check(native.lib().lz4b200_encode_batch(self._h, src, src_off, src_len, dst, dst_off, dst_cap, out_len, int(n),
                                                       native.MODE_HC if hc else native.MODE_FAST,
                                                       self._mem(device, mem), stream), "encode_batch")

    def decode_batch_ptr(self, src, src_off, src_len, dst, dst_off, dst_cap, out_len, n, known=True, device=True, stream=0, mem=None):
        native.check(native.lib().lz4b200_decode_batch(self._h, src, src_off, src_len, dst, dst_off, dst_cap, out_len, int(n),
                                                       1 if known else 0, self._mem(device, mem), stream), "decode_batch")

    def measure_batch_ptr(self, src, src_off, src_len, dst_cap, out_len, n, known=False, device=True, stream=0):
        native.check(native.lib().lz4b200_measure_batch(self._h, src, src_off, src_len, dst_cap, out_len, int(n), 1 if known else 0,
                                                        native.MEM_DEVICE if device else native.MEM_HOST, stream), "measure_batch")

    def encode_batch_packed_ptr(self, src, src_off, src_len, dst_cap, dst, dst_total_cap, out_off, out_len, n, hc=False):
        native.check(native.lib().lz4b200_encode_batch_packed(self._h, src, src_off, src_len, dst_cap, dst, int(dst_total_cap),
                                                              out_off, out_len, int(n),
                                                              native.MODE_HC if hc else native.MODE_FAST), "encode_batch_packed")

    def encode_blocks_packed(self, blocks, caps=None, hc=False):
        """Host batch with packed output.  Returns (out_len list, out_off list[n+1], packed bytes)."""
        n = len(blocks)
        src, lens, src_off = _pack(blocks)
        caps = np.array([native.lib().lz4b200_compress_bound(int(l)) for l in lens] if caps is None else caps, np.int32)
        total_cap = int(caps.sum())
        dst = np.full(total_cap + 16, 0xEE, np.uint8)
        out = np.zeros(n, np.int32); off = np.zeros(n + 1, np.int64)
        self.encode_batch_packed_ptr(src.ctypes.data, src_off.ctypes.data, lens.ctypes.data, caps.ctypes.data, dst.ctypes.data,
                                     total_cap, off.ctypes.data, out.ctypes.data, n, hc=hc)
        assert (dst[int(off[n]):] == 0xEE).all(), "packed encode wrote past the reported total"
        return out.tolist(), off.tolist(), dst[:int(off[n])].tobytes()

    # ---- numpy (host memory) convenience -----------------------------------------------------------------------
    def encode_blocks(self, blocks, caps=None, hc=False):
        """blocks: list of bytes-like.  Returns (out_len list, list of bytes) -- one host-memory batch call."""
        n = len(blocks)
        src, lens, src_off = _pack(blocks)
        caps = np.array([native.lib().lz4b200_compress_bound(int(l)) for l in lens] if caps is None else caps, np.int32)
        dst_off = _offsets(caps)
        dst = np.full(int(caps.sum()) + 16, 0xEE, np.uint8)
        out = np.zeros(n, np.int32)
        if n:
            self.encode_batch_ptr(src.ctypes.data, src_off.ctypes.data, lens.ctypes.data, dst.ctypes.data, dst_off.ctypes.data,
                                  caps.ctypes.data, out.ctypes.data, n, hc=hc, device=False)
        return out.tolist(), [dst[int(o):int(o) + max(int(r), 0)].tobytes() for o, r in zip(dst_off, out)]

    def decode_blocks(self, blocks, caps, known=True):
        n = len(blocks)
        src, lens, src_off = _pack(blocks)
        caps = np.array(caps, np.int32)
        dst_off = _offsets(caps)
        dst = np.zeros(int(caps.sum()) + 16, np.uint8)
        out = np.zeros(n, np.int32)
        if n:
            self.decode_batch_ptr(src.ctypes.data, src_off.ctypes.data, lens.ctypes.data, dst.ctypes.data, dst_off.ctypes.data,
                                  caps.ctypes.data, out.ctypes.data, n, known=known, device=False)
        res = out.tolist()
        outs = []
        for o, c, r in zip(dst_off, caps, res):
            m = int(c) if known else max(int(r), 0)
            outs.append(dst[int(o):int(o) + m].tobytes())
        return res, outs

    def decode_blocks_to_device(self, blocks, out):
        """Raw LZ4 blocks (bytes-like) whose decoded sizes nobody stored, decoded back to back into the bytes of a contiguous
        CUDA tensor: one lz4b200_decode_batch_packed_to_device call, the compressed bytes cross PCIe once.  Returns
        (out_len list, out_off list[n+1]): block i lies at out_off[i], out_off[n] is the total.  When the total exceeds the
        tensor's size its bytes are unspecified and out_len holds the sizes: allocate out_off[n] bytes and call again.  A
        malformed block has a negative out_len and occupies no bytes."""
        from . import batch
        n = len(blocks)
        src, lens, src_off = _pack(blocks)
        out_len, out_off = np.zeros(n, np.int32), np.zeros(n + 1, np.int64)
        batch.decode_from_host_packed(self, src, src_off, lens, batch._flat_bytes(out), out_off, out_len)
        return out_len.tolist(), out_off.tolist()

    def measure_blocks(self, blocks, caps=None, known=False):
        """What decode_blocks(blocks, caps, known) would return as out_len, without decoding: one host-memory batch call.
        caps=None (unknown size only): no limit on the decoded size (INT32_MAX per block)."""
        if caps is None and known:
            raise ValueError("known-size measuring needs the decoded sizes (caps)")
        n = len(blocks)
        src, lens, src_off = _pack(blocks)
        caps = None if caps is None else np.array(caps, np.int32)
        out = np.zeros(n, np.int32)
        if n:
            self.measure_batch_ptr(src.ctypes.data, src_off.ctypes.data, lens.ctypes.data, None if caps is None else caps.ctypes.data,
                                   out.ctypes.data, n, known=known, device=False)
        return out.tolist()

    # ---- framing ----------------------------------------------------------------------------------------------
    def stream_encode(self, data: bytes, block_size: int = 1 << 20, high_compression: bool = False) -> bytes:
        """The bytes LZ4Stream(inner, Compress, highCompression, blockSize) emits for Write(data); Close()."""
        l = native.lib()
        src = np.frombuffer(bytes(data) + b"\0", np.uint8)
        cap = int(l.lz4b200_stream_bound(len(data), block_size))
        dst = np.zeros(cap + 16, np.uint8)
        w = l.lz4b200_stream_encode(self._h, src.ctypes.data, len(data), block_size, int(high_compression), dst.ctypes.data, cap)
        if w < 0:
            raise native.Lz4B200Error(f"stream_encode failed ({w}): {native.last_error()}")
        return dst[:w].tobytes()

    def stream_decode(self, data: bytes) -> bytes:
        l = native.lib()
        src = np.frombuffer(bytes(data) + b"\0", np.uint8)
        total = int(l.lz4b200_stream_decoded_size(src.ctypes.data, len(data)))
        if total < 0:
            raise EOFError("LZ4Stream: unexpected end of stream / corrupt chunk header")     # EndOfStreamException
        dst = np.zeros(total + 16, np.uint8)
        r = l.lz4b200_stream_decode(self._h, src.ctypes.data, len(data), dst.ctypes.data, total)
        if r == native.E_FORMAT:
            raise ValueError("LZ4 block has been corrupted")
        if r < 0:
            raise native.Lz4B200Error(f"stream_decode failed ({r}): {native.last_error()}")
        return dst[:total].tobytes()

    def stream_encode_from_device(self, raw, block_size: int = 1 << 20, high_compression: bool = False) -> bytes:
        """stream_encode of a contiguous CUDA tensor's bytes, written straight from device memory
        (lz4b200_stream_encode_from_device)."""
        from . import batch
        return batch.stream_encode_to_host(self, raw, block_size, high_compression).tobytes()

    def stream_decode_to_device(self, data: bytes, out) -> int:
        """stream_decode into the first bytes of a contiguous CUDA tensor (lz4b200_stream_decode_to_device); returns the
        decoded size.  Raises like stream_decode, and Lz4B200Error when `out` is too small."""
        from . import batch
        src = np.frombuffer(bytes(data) + b"\0", np.uint8)
        if native.lib().lz4b200_stream_decoded_size(src.ctypes.data, len(data)) < 0:
            raise EOFError("LZ4Stream: unexpected end of stream / corrupt chunk header")     # EndOfStreamException
        try:
            return batch.stream_decode_to_device(self, src[:len(data)], out)
        except native.Lz4B200Error as e:
            if f"status {native.E_FORMAT}:" in str(e):
                raise ValueError("LZ4 block has been corrupted") from e
            raise


def _is_tensor(x) -> bool:
    """A torch tensor (without importing torch when the caller has not)."""
    torch = sys.modules.get("torch")
    return torch is not None and isinstance(x, torch.Tensor)


def _tensor_bytes(t):
    """The bytes of a contiguous tensor in storage order, as a flat uint8 tensor on the same memory."""
    if not t.is_contiguous():
        raise TypeError("expected a contiguous tensor")
    import torch
    return t.reshape(-1).view(torch.uint8)


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        dev = 0
        try:
            import torch
            if torch.cuda.is_available():
                dev = torch.cuda.current_device()
        except Exception:
            pass
        _default_ctx = Context(dev)
    return _default_ctx


class CudaLZ4Service:
    """ILZ4Service (src/LZ4/ILZ4Service.cs:30-36) over the single-block C entry points."""

    CodecName = "CUDA sm_90a"

    @staticmethod
    def _ptr(buf, offset):
        a = np.frombuffer(buf, np.uint8) if not isinstance(buf, np.ndarray) else buf
        return a, a.ctypes.data + offset

    def Encode(self, input, inputOffset, inputLength, output, outputOffset, outputLength) -> int:
        _, sp = self._ptr(input, inputOffset)
        _, dp = self._ptr(output, outputOffset)
        return int(native.lib().lz4b200_compress_limitedOutput(sp, dp, inputLength, outputLength))

    def EncodeHC(self, input, inputOffset, inputLength, output, outputOffset, outputLength) -> int:
        _, sp = self._ptr(input, inputOffset)
        _, dp = self._ptr(output, outputOffset)
        r = int(native.lib().lz4b200_compressHC_limitedOutput(sp, dp, inputLength, outputLength))
        return r if r > 0 else -1                                    # src/LZ4ps/LZ4Codec.Safe.cs:721-723

    def Decode(self, input, inputOffset, inputLength, output, outputOffset, outputLength, knownOutputLength) -> int:
        _, sp = self._ptr(input, inputOffset)
        _, dp = self._ptr(output, outputOffset)
        if knownOutputLength:
            r = int(native.lib().lz4b200_uncompress(sp, dp, inputLength, outputLength))
            if r != inputLength:                                     # src/LZ4ps/LZ4Codec.Safe.cs:539-542
                raise ValueError("LZ4 block is corrupted, or invalid length has been given.")
            return outputLength
        r = int(native.lib().lz4b200_uncompress_unknownOutputSize(sp, dp, inputLength, outputLength))
        if r < 0:                                                    # :546-549
            raise ValueError("LZ4 block is corrupted, or invalid length has been given.")
        return r


class LZ4Codec:
    """Static facade, src/LZ4/LZ4Codec.cs.  Buffers are bytearray / numpy uint8 arrays (the byte[] of the original)."""

    _service = CudaLZ4Service()
    CodecName = "CUDA sm_90a/CUDA sm_90a/CUDA sm_90aHC"

    @staticmethod
    def MaximumOutputLength(inputLength: int) -> int:                # :313-316
        return inputLength + inputLength // 255 + 16

    @staticmethod
    def _check(buf, offset, length, what):                           # src/LZ4ps/LZ4Codec.cs:151-170
        if buf is None:
            raise TypeError(f"{what} is null")
        if length < 0:
            length = len(buf) - offset
        if offset < 0 or offset + length > len(buf):
            raise ValueError(f"{what}Offset and {what}Length are invalid for given {what}")
        return length

    @classmethod
    def Encode(cls, input, inputOffset=0, inputLength=-1, output=None, outputOffset=0, outputLength=-1):
        if output is None:                                           # byte[] Encode(byte[], int, int)  :344-365
            inputLength = cls._check(input, inputOffset, inputLength, "input")
            if inputLength == 0:
                return bytes()
            out = bytearray(cls.MaximumOutputLength(inputLength))
            n = cls.Encode(input, inputOffset, inputLength, out, 0, len(out))
            if n < 0:
                raise ValueError("Compression has been corrupted")
            return bytes(out[:n])
        inputLength = cls._check(input, inputOffset, inputLength, "input")
        outputLength = cls._check(output, outputOffset, outputLength, "output")
        if inputLength == 0 or outputLength == 0:
            return 0
        return cls._service.Encode(input, inputOffset, inputLength, output, outputOffset, outputLength)

    @classmethod
    def EncodeHC(cls, input, inputOffset=0, inputLength=-1, output=None, outputOffset=0, outputLength=-1):
        if output is None:
            inputLength = cls._check(input, inputOffset, inputLength, "input")
            if inputLength == 0:
                return bytes()
            out = bytearray(cls.MaximumOutputLength(inputLength))
            n = cls.EncodeHC(input, inputOffset, inputLength, out, 0, len(out))
            if n < 0:
                raise ValueError("Compression has been corrupted")
            return bytes(out[:n])
        inputLength = cls._check(input, inputOffset, inputLength, "input")
        outputLength = cls._check(output, outputOffset, outputLength, "output")
        if inputLength == 0 or outputLength == 0:
            return 0 if inputLength == 0 else -1
        return cls._service.EncodeHC(input, inputOffset, inputLength, output, outputOffset, outputLength)

    @classmethod
    def Decode(cls, input, inputOffset, inputLength, output=None, outputOffset=0, outputLength=0, knownOutputLength=False):
        if output is None or isinstance(output, int):                # byte[] Decode(byte[], int, int, int outputLength)  :448-462
            want = outputOffset if output is None else output
            inputLength = cls._check(input, inputOffset, inputLength, "input")
            if inputLength == 0:
                return bytes()
            out = bytearray(want)
            n = cls.Decode(input, inputOffset, inputLength, out, 0, want, True)
            if n != want:
                raise ValueError("outputLength is not valid")
            return bytes(out)
        cuda = _is_tensor(output) and output.is_cuda                 # its bytes in storage order; offset and length count bytes
        if cuda:
            if knownOutputLength:
                raise TypeError("a CUDA tensor output takes knownOutputLength=False")
            output = _tensor_bytes(output)
        inputLength = cls._check(input, inputOffset, inputLength, "input")
        outputLength = cls._check(output, outputOffset, outputLength, "output")
        if inputLength == 0 or outputLength == 0:                    # CheckArguments :156-160 + `if (outputLength == 0) return 0` (Safe.cs:470)
            return 0
        if cuda:                                                     # decoded straight into device memory
            block = bytes(input[inputOffset:inputOffset + inputLength])
            res, off = default_context().decode_blocks_to_device([block], output[outputOffset:outputOffset + outputLength])
            if res[0] < 0 or off[1] > outputLength:                  # src/LZ4ps/LZ4Codec.Safe.cs:546-549
                raise ValueError("LZ4 block is corrupted, or invalid length has been given.")
            return res[0]
        return cls._service.Decode(input, inputOffset, inputLength, output, outputOffset, outputLength, knownOutputLength)

    # ---- Wrap / Unwrap (:510-599) ------------------------------------------------------------------------------
    # Wrap / WrapHC also take a contiguous CUDA tensor (its bytes in storage order; offset and length count bytes): the
    # packet is written straight from device memory (lz4b200_wrap_batch_packed_from_device), the same bytes as for the
    # tensor's host copy.
    @staticmethod
    def _wrap(data, hc):
        if _is_tensor(data) and data.numel():                        # (an empty input has no device address to read)
            from . import batch
            n = data.numel()
            dst = np.empty(n + 8, np.uint8)
            off, out = np.zeros(2, np.int64), np.zeros(1, np.int32)
            w = batch.wrap_to_host_packed(default_context(), data, np.zeros(1, np.int64), np.array([n], np.int32), dst, off, out,
                                          hc=hc)
            return dst[:w].tobytes()
        l = native.lib()
        src = np.frombuffer(bytes(data) + b"\0", np.uint8)
        dst = np.zeros(len(data) + 8 + 16, np.uint8)
        r = l.lz4b200_wrap(default_context().handle, src.ctypes.data, len(data), int(hc), dst.ctypes.data, len(data) + 8)
        if r < 0:
            raise native.Lz4B200Error(f"wrap failed ({r}): {native.last_error()}")
        return dst[:r].tobytes()

    @staticmethod
    def _wrap_input(inputBuffer, inputOffset, inputLength):
        """The input of Wrap / WrapHC: bytes, or the flat uint8 view of a CUDA tensor's bytes."""
        cuda = _is_tensor(inputBuffer) and inputBuffer.is_cuda
        if cuda:
            inputBuffer = _tensor_bytes(inputBuffer)
        inputLength = min(len(inputBuffer) - inputOffset, inputLength)
        if inputLength < 0:
            raise ValueError("inputBuffer size of inputLength is invalid")
        part = inputBuffer[inputOffset:inputOffset + inputLength]
        return part if cuda else bytes(part)

    @classmethod
    def Wrap(cls, inputBuffer, inputOffset=0, inputLength=2 ** 31 - 1):
        return cls._wrap(cls._wrap_input(inputBuffer, inputOffset, inputLength), False)

    @classmethod
    def WrapHC(cls, inputBuffer, inputOffset=0, inputLength=2 ** 31 - 1):
        return cls._wrap(cls._wrap_input(inputBuffer, inputOffset, inputLength), True)

    @staticmethod
    def Unwrap(inputBuffer, inputOffset=0):
        l = native.lib()
        data = bytes(inputBuffer[inputOffset:])
        src = np.frombuffer(data + b"\0", np.uint8)
        size = l.lz4b200_unwrap_size(src.ctypes.data, len(data))
        if size < 0:
            raise ValueError("inputBuffer size is invalid or has been corrupted")
        dst = np.zeros(size + 16, np.uint8)
        r = l.lz4b200_unwrap(default_context().handle, src.ctypes.data, len(data), dst.ctypes.data, size)
        if r < 0:
            raise ValueError("LZ4 block is corrupted, or invalid length has been given.")
        return dst[:r].tobytes()


def wrap_batch(inputs, hc=False, ctx=None):
    """n packets in ONE encode batch (lz4b200_wrap_batch): packet i == LZ4Codec.Wrap / WrapHC of inputs[i]
    (src/LZ4/LZ4Codec.cs:510-543).  Returns a list of bytes."""
    ctx = ctx or default_context()
    n = len(inputs)
    src, lens, so = _pack(inputs)
    caps = lens + 8
    do = _offsets(caps)
    dst = np.zeros(int(caps.sum()) + 16, np.uint8)
    out = np.zeros(n, np.int32)
    native.check(native.lib().lz4b200_wrap_batch(ctx.handle, src.ctypes.data, so.ctypes.data, lens.ctypes.data, int(hc),
                                                 dst.ctypes.data, do.ctypes.data, caps.ctypes.data, out.ctypes.data, n), "wrap_batch")
    return [dst[int(o):int(o) + int(r)].tobytes() for o, r in zip(do, out)]


def unwrap_batch(packets, ctx=None):
    """Mirror image (lz4b200_unwrap_batch, src/LZ4/LZ4Codec.cs:574-599).  Raises ValueError on a corrupt packet."""
    ctx = ctx or default_context()
    n = len(packets)
    l = native.lib()
    src, lens, so = _pack(packets)
    sizes = np.array([l.lz4b200_unwrap_size(src.ctypes.data + int(o), int(k)) for o, k in zip(so, lens)], np.int32)
    if (sizes < 0).any():
        raise ValueError("inputBuffer size is invalid or has been corrupted")
    do = _offsets(sizes)
    dst = np.zeros(int(sizes.sum()) + 16, np.uint8)
    out = np.zeros(n, np.int32)
    native.check(l.lz4b200_unwrap_batch(ctx.handle, src.ctypes.data, so.ctypes.data, lens.ctypes.data, dst.ctypes.data,
                                        do.ctypes.data, sizes.ctypes.data, out.ctypes.data, n), "unwrap_batch")
    if (out < 0).any():
        raise ValueError("LZ4 block is corrupted, or invalid length has been given.")
    return [dst[int(o):int(o) + int(r)].tobytes() for o, r in zip(do, out)]


class LZ4StreamMode:
    Compress, Decompress = 0, 1                                       # src/LZ4/LZ4StreamMode.cs


class LZ4StreamFlags:
    None_, InteractiveRead, HighCompression, IsolateInnerStream, Default = 0, 1, 2, 4, 0    # src/LZ4/LZ4StreamFlags.cs


class LZ4Stream:
    """``LZ4Stream`` (src/LZ4/LZ4Stream.cs) over a Python binary file object.

    Wire format and chunk boundaries are the reference's (a chunk per ``blockSize`` bytes written, a partial chunk on
    ``Flush``/``Close``, FlushCurrentChunk :239-269); the dispatcher differs: up to ``batchBlocks`` buffered blocks (and at
    most ``maxBufferBytes``) are encoded / decoded by ONE batched GPU call instead of one block per call.  With
    ``InteractiveRead`` the reader decodes every chunk as soon as it has been read, like the reference (:376-401): a
    socket or pipe that has delivered one chunk is never asked for the next one before the caller has seen the first.

    ``Write`` also takes a contiguous CUDA tensor (its bytes in storage order) and ``ReadInto`` fills one: whole blocks are
    encoded straight from device memory and whole chunks decoded straight into it (the context's
    ``stream_encode_from_device`` / ``stream_decode_to_device``), so the raw bytes never cross PCIe.  The wire bytes and
    chunk boundaries are those of the same bytes written from host memory."""

    def __init__(self, innerStream, compressionMode, compressionFlags=LZ4StreamFlags.Default, blockSize=1024 * 1024,
                 batchBlocks=256, context: Optional[Context] = None, maxBufferBytes=64 * 1024 * 1024):
        self._inner = innerStream
        self._mode = compressionMode
        self._hc = bool(compressionFlags & LZ4StreamFlags.HighCompression)
        self._interactive = bool(compressionFlags & LZ4StreamFlags.InteractiveRead)
        self._isolate = bool(compressionFlags & LZ4StreamFlags.IsolateInnerStream)
        self._block = max(16, int(blockSize))                          # :131,138
        self._batch = max(1, int(batchBlocks))
        # write buffer cap (whole blocks, at least one) / read-ahead cap (whole chunks, at least one: blockSize is the WRITER's)
        self._max_bytes = max(self._block if compressionMode == LZ4StreamMode.Compress else 1, int(maxBufferBytes))
        self._ctx = context or default_context()
        self._pending = bytearray()
        self._ready = b""
        self._rpos = 0
        self._closed = False

    CanSeek = False

    @property
    def CanRead(self):
        return self._mode == LZ4StreamMode.Decompress

    @property
    def CanWrite(self):
        return self._mode == LZ4StreamMode.Compress

    # ---- write side (:444-470) ----
    def Write(self, buffer, offset=0, count=None):
        if not self.CanWrite:
            raise NotImplementedError("Operation 'Write' is not supported")
        if _is_tensor(buffer):
            self._write_tensor(buffer, offset, count)
            return
        count = len(buffer) - offset if count is None else count
        self._pending += bytes(buffer[offset:offset + count])
        self._drain()

    def _drain(self):
        full = min(self._batch, self._max_bytes // self._block) * self._block
        while len(self._pending) > full:          # a full buffer is flushed only when more data arrives (:463-467)
            self._emit(full)

    def _write_tensor(self, tensor, offset, count):
        """Bytes [offset, offset + count) of a tensor: the head that completes the pending chunk comes to the host (less
        than one block), the whole blocks after it are encoded from device memory, the tail (less than one block) stays
        pending.  The chunks are the ones a host write of the same bytes makes."""
        t = _tensor_bytes(tensor)
        count = t.numel() - offset if count is None else count
        if offset < 0 or count < 0 or offset + count > t.numel():
            raise ValueError("offset and count are invalid for the given buffer")
        t = t[offset:offset + count]
        head = min(count, -len(self._pending) % self._block)
        self._pending += t[:head].cpu().numpy().tobytes()
        whole = (count - head) // self._block * self._block
        if whole:
            if self._pending:                     # whole blocks only: the same chunks as one host write
                self._emit(len(self._pending))
            self._inner.write(self._ctx.stream_encode_from_device(t[head:head + whole], self._block, self._hc))
        self._pending += t[head + whole:].cpu().numpy().tobytes()
        self._drain()

    def WriteByte(self, value):
        self.Write(bytes([value]))

    def _emit(self, n):
        self._inner.write(self._ctx.stream_encode(bytes(self._pending[:n]), self._block, self._hc))
        del self._pending[:n]

    def Flush(self):                                                    # :337-340
        if self.CanWrite and self._pending:
            self._emit(len(self._pending))

    def Close(self):                                                    # Dispose :472-478
        if not self._closed:
            self.Flush()
            self._closed = True
            if not self._isolate and hasattr(self._inner, "close"):
                self._inner.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.Close()

    # ---- read side (:376-401, AcquireNextChunk :274-312) ----
    def _read_varint(self, raw, first):
        v, count = 0, 0
        while True:
            b = self._inner.read(1)
            if not b:
                if first and count == 0:
                    return None
                raise EOFError("Unexpected end of stream")
            raw += b
            v += (b[0] & 0x7F) << count
            count += 7
            if not (b[0] & 0x80) or count >= 64:
                return v

    def _acquire(self, out=None, room=0):
        """Reads the next chunks.  With `out` (a flat uint8 tensor), the leading chunks whose decoded bytes fit in `room`
        are decoded straight into it; the rest are decoded to the host as without it.  Returns None at the end of the
        stream, else the number of bytes decoded into `out`."""
        raw = bytearray()
        direct = b""
        decoded = 0
        for _ in range(1 if self._interactive else self._batch):       # interactive: one chunk, then hand it over
            start = len(raw)
            flags = self._read_varint(raw, True)
            if flags is None:
                break
            raw_len = self._read_varint(raw, False)
            comp_len = self._read_varint(raw, False) if flags & 1 else raw_len
            if comp_len > raw_len or raw_len > 0x7FFFFFFF:
                raise EOFError("Unexpected end of stream")             # :288 corrupted (lengths are ints in the reference)
            payload = self._inner.read(comp_len)
            while len(payload) < comp_len:                              # ReadBlock :205-221: no partial chunks
                more = self._inner.read(comp_len - len(payload))
                if not more:
                    raise EOFError("Unexpected end of stream")
                payload += more
            raw += payload
            if out is not None and start == 0 and decoded + raw_len <= room:
                direct += raw                                           # every chunk so far fits: it goes to the device
                del raw[:]
            decoded += raw_len
            if decoded >= self._max_bytes:                              # cap the read-ahead by bytes, not only by chunks
                break
        if not raw and not direct:
            return None
        self._ready = self._ctx.stream_decode(bytes(raw)) if raw else b""
        self._rpos = 0
        return self._ctx.stream_decode_to_device(bytes(direct), out) if direct else 0

    def Read(self, count):
        """Returns up to `count` bytes (b"" at end of stream); with InteractiveRead returns as soon as it has any."""
        if not self.CanRead:
            raise NotImplementedError("Operation 'Read' is not supported")
        out = bytearray()
        while count > 0:
            chunk = min(count, len(self._ready) - self._rpos)
            if chunk > 0:
                out += self._ready[self._rpos:self._rpos + chunk]
                self._rpos += chunk
                if self._interactive:
                    break
                count -= chunk
            elif self._acquire() is None:
                break
        return bytes(out)

    def ReadInto(self, tensor):
        """Read into a contiguous CUDA tensor's bytes, up to its size: returns the bytes read (0 at end of stream), with
        Read's semantics (InteractiveRead included).  Bytes already decoded come first; chunks that fit in what is left are
        decoded straight into the tensor; the chunk that straddles its end is decoded to the host, like Read."""
        if not self.CanRead:
            raise NotImplementedError("Operation 'Read' is not supported")
        out = _tensor_bytes(tensor)
        import torch
        count, pos = out.numel(), 0
        while pos < count:
            chunk = min(count - pos, len(self._ready) - self._rpos)
            if chunk > 0:
                part = np.frombuffer(self._ready, np.uint8, chunk, self._rpos)
                out[pos:pos + chunk].copy_(torch.from_numpy(part.copy()))
                self._rpos += chunk
                pos += chunk
                if self._interactive:
                    break
                continue
            got = self._acquire(out[pos:], count - pos)
            if got is None:
                break
            pos += got
            if got and self._interactive:
                break
        return pos

    def ReadByte(self):
        b = self.Read(1)
        return b[0] if b else -1
