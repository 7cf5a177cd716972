// lz4_stream.cuh -- the LZ4Stream chunk frame (src/LZ4/LZ4Stream.cs:239-269) written and read on the device, for every
// stream call (capi.cu stream_encode / stream_decode: host or device raw bytes, stream bytes in host memory).
//
// A chunk is  varint(flags) varint(rawLen) [varint(compLen)] payload : the compressed bytes, or the raw bytes when the
// encoder's result r (at capacity = rawLen) does not satisfy 0 < r < rawLen (:248-255).  flags = compressed (1) | HC (2);
// the HC bit is set on stored chunks too (:257-264).  The stream bytes live in host memory and the host walks their
// headers (framing.cpp stream_walk); the device writes the frames of an encode and copies the stored payloads of a
// decode:
//   encode:  encode (capacity = chunk length) -> frame sizes (a thread per chunk) -> scan (launch_compact without a
//            payload) -> frame write (a warp per chunk: header bytes, then the payload from the encoder's slot or, for a
//            stored chunk, from the source: the caller's device memory, or the pipeline's staged copy of host bytes)
//   decode:  known-size decode of the compressed chunks (stored ones get the neutral entry, see lz4_wrap.cuh) -> stored
//            copy (a warp per chunk: a stored chunk's payload to its place in the output; compressed chunks do nothing)
// The asynchronous calls add two per-thread rules: the encode's chunk table, computed on the device (stream_cut_one), and
// the decode's status, kept on the device (stream_chunk_failed).
// This is the library's only writer of the format.
#pragma once
#include "lz4_copy.cuh"

namespace lz4b200 {

constexpr int32_t STREAM_FLAG_COMPRESSED = 1, STREAM_FLAG_HC = 2;     // ChunkFlags, LZ4Stream.cs:43-58
constexpr int32_t STREAM_HEADER_MAX = 11;                             // flags (1 byte) + two varints of <= 5 bytes

SIMT_DEV int stream_varint_size(uint32_t v) { return v < (1u << 7) ? 1 : v < (1u << 14) ? 2 : v < (1u << 21) ? 3 : v < (1u << 28) ? 4 : 5; }

// the chunk is compressed when the encoder's result shrinks it (LZ4Stream.cs:248-255)
SIMT_DEV bool stream_compressed(int32_t raw, int32_t r) { return r > 0 && r < raw; }

SIMT_DEV int32_t stream_header_size(int32_t raw, int32_t r)
{
    return 1 + stream_varint_size((uint32_t)raw) + (stream_compressed(raw, r) ? stream_varint_size((uint32_t)r) : 0);
}

// bytes of the chunk's frame: header + payload (<= raw + STREAM_HEADER_MAX)
SIMT_DEV int32_t stream_frame_size(int32_t raw, int32_t r)
{
    return stream_header_size(raw, r) + (stream_compressed(raw, r) ? r : raw);
}

// byte j of varint(v) (LZ4Stream.cs:225-236), j < stream_varint_size(v)
SIMT_DEV uint8_t stream_varint_byte(uint32_t v, int j)
{
    return (uint8_t)(((v >> (7 * j)) & 0x7Fu) | (j + 1 < stream_varint_size(v) ? 0x80u : 0u));
}

// byte k of the chunk's header, k < stream_header_size(raw, r)
SIMT_DEV uint8_t stream_header_byte(int32_t raw, int32_t r, bool hc, int k)
{
    const bool comp = stream_compressed(raw, r);
    if (k == 0) return (uint8_t)((comp ? STREAM_FLAG_COMPRESSED : 0) | (hc ? STREAM_FLAG_HC : 0));
    const int lr = stream_varint_size((uint32_t)raw);
    return k <= lr ? stream_varint_byte((uint32_t)raw, k - 1) : stream_varint_byte((uint32_t)r, k - 1 - lr);
}

// Frame write, called by all 32 lanes of a warp with the same arguments: the frame of a chunk of `raw` bytes at `in`
// whose encoder result is r and compressed bytes are at `comp`, written at `frame`.  Lanes below the header length each
// write one header byte; the payload is copied by the whole warp.  Returns the frame's size.
SIMT_DEV int32_t stream_frame_one(const uint8_t* in, int32_t raw, const uint8_t* comp, int32_t r, bool hc, uint8_t* frame, int lane)
{
    const int32_t h = stream_header_size(raw, r);
    if (lane < h) simt::stg_u8(frame + lane, stream_header_byte(raw, r, hc, lane));
    const bool c = stream_compressed(raw, r);
    const int32_t len = c ? r : raw;
    if (len > 0) {
        const InputSrc s{c ? comp : in};
        group_copy<32, false>(frame + h, s, (uint32_t)len, lane, 0xFFFFFFFFu);
    }
    return h + len;
}

// Stored copy, called by all 32 lanes of a warp with the same arguments: a stored chunk's payload (`stored` bytes at
// `payload`) to its place `dst` in the output.  stored = 0 (a compressed chunk) does nothing.
SIMT_DEV void stream_stored_one(const uint8_t* payload, int32_t stored, uint8_t* dst, int lane)
{
    if (stored <= 0) return;
    const InputSrc s{payload};
    group_copy<32, false>(dst, s, (uint32_t)stored, lane, 0xFFFFFFFFu);
}

// The asynchronous encode (capi.cu run_async) holds no per-chunk host metadata: each stage's chunk table is computed on
// the device.  Entry i of the stage whose first chunk is `first`, in a stream of n bytes cut into block_size chunks: the
// chunk is bytes [so, so + len) of the source, encoded into the stage's dense slot at dof with capacity cap = len.  Only
// a stream's last chunk is short, so slot i starts at i * block_size.
SIMT_DEV void stream_cut_one(int64_t i, int64_t first, int32_t block_size, int64_t n, int64_t* so, int32_t* len, int64_t* dof,
                             int32_t* cap)
{
    const int64_t at = (first + i) * block_size;
    const int32_t l = (int32_t)(n - at < block_size ? n - at : block_size);
    so[i] = at; len[i] = l; dof[i] = i * (int64_t)block_size; cap[i] = l;
}

// The decode's status rule: an entry fails when it is a compressed chunk (stored == 0: no stored payload) whose known-size
// decode did not read exactly its compLen bytes (res, negative for a malformed block; LZ4Codec.Safe.cs:539-542).  Stored
// chunks are copied, never decoded, and never fail.
SIMT_DEV bool stream_chunk_failed(int32_t stored, int32_t comp_len, int32_t res) { return stored == 0 && res != comp_len; }

}  // namespace lz4b200
