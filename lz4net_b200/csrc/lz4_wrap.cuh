// lz4_wrap.cuh -- the Wrap / Unwrap packet (src/LZ4/LZ4Codec.cs:510-543, 574-599) around the batch codec, on the device.
//
// A packet is  u32le rawLen, u32le storedLen, payload : the compressed bytes, or the input itself when compression does not
// shrink it (storedLen == rawLen).  The device entry points (capi.cu lz4b200_wrap_batch_device / unwrap_batch_device /
// unwrap_batch_packed) run the existing encoders and decoders unchanged between a prep and a finish step per packet:
//   wrap:    prep (a thread per packet: the encoder's view of the batch, payload at dst_off + 8 with capacity = the input
//            length) -> encode -> finish (a warp per packet: header, stored-raw rule, stored copy)
//   unwrap:  prep (a thread per packet: the header, bounded by the packet's length; a decode entry for compressed packets, a
//            neutral one otherwise) -> known-size decode -> finish (a warp per packet: stored copy, status)
// A neutral decode entry (src_len 0, dst_cap 0) reads and writes nothing in every decoder: they all reject an empty stream
// before touching it (decode_block / decode_block_staged / lpb_decode_warp: isize <= 0), and only their result, which
// the finish step ignores, is stored.
// The wrap side is the library's only writer of the packet: the calls with a side in host memory (capi.cu wrap_packets)
// run the same prep and finish inside the host pipeline.  Those unwraps read the headers on the host (framing.cpp
// read_header, the same rules as unwrap_header) and reuse the stored copy of lz4_stream.cuh.
#pragma once
#include "lz4_copy.cuh"

namespace lz4b200 {

constexpr int32_t WRAP_HEADER = 8;
constexpr int32_t WRAP_E_ARG = -1, WRAP_E_FORMAT = -5;           // LZ4B200_E_ARG / LZ4B200_E_FORMAT

// ---- wrap -----------------------------------------------------------------------------------------------------------
// The packet is valid when its input length is not negative (LZ4Codec.cs:513-514) and its capacity holds input + header.
SIMT_DEV bool wrap_valid(int32_t len, int32_t cap) { return len >= 0 && (int64_t)cap >= (int64_t)len + WRAP_HEADER; }

// Prep: what the encoder sees of packet i.  An invalid packet, or an empty input, is given nothing to read and capacity 0,
// so the encoder reads and writes nothing for it.
SIMT_DEV void wrap_prep_one(int64_t dst_off, int32_t len, int32_t cap, int64_t* enc_off, int32_t* enc_len, int32_t* enc_cap)
{
    const bool go = wrap_valid(len, cap) && len > 0;
    *enc_off = dst_off + WRAP_HEADER;
    *enc_len = go ? len : 0;
    *enc_cap = go ? len : 0;
}

// Stored unless compression shrinks the input (LZ4Codec.cs:527-540).  r = the encoder's result.
SIMT_DEV int32_t wrap_stored(int32_t len, int32_t r) { return r >= len || r <= 0 ? len : r; }

// Finish, called by all 32 lanes of a warp with the same arguments: writes the header (and, for a stored packet, the input
// over the payload) and returns the packet's out_len.  An invalid packet gets LZ4B200_E_ARG and nothing is written.
SIMT_DEV int32_t wrap_finish_one(const uint8_t* in, int32_t len, int32_t cap, int32_t r, uint8_t* pkt, int lane)
{
    if (!wrap_valid(len, cap)) return WRAP_E_ARG;
    const int32_t stored = wrap_stored(len, len > 0 ? r : 0);
    if (lane < WRAP_HEADER) {
        const uint32_t v = lane < 4 ? (uint32_t)len : (uint32_t)stored;
        simt::stg_u8(pkt + lane, (uint8_t)(v >> (8 * (lane & 3))));
    }
    if (stored == len && len > 0) {
        const InputSrc s{in};
        group_copy<32, false>(pkt + WRAP_HEADER, s, (uint32_t)len, lane, 0xFFFFFFFFu);
    }
    return stored + WRAP_HEADER;
}

// ---- unwrap ---------------------------------------------------------------------------------------------------------
// The packet header (LZ4Codec.cs:574-599): the unwrapped size, or LZ4B200_E_FORMAT.  The header is read only when the packet holds
// it, byte by byte: a packet shorter than 8 bytes, or one at any alignment, never reads a byte outside itself.
SIMT_DEV int32_t unwrap_header(const uint8_t* p, int32_t n, int32_t* raw, int32_t* stored)
{
    if (n < WRAP_HEADER) return WRAP_E_FORMAT;                                          // LZ4Codec.cs:577-578
    uint32_t h[2] = {0, 0};
    for (int k = 0; k < WRAP_HEADER; k++) h[k >> 2] |= (uint32_t)simt::ldg_nc_u8(p + k) << (8 * (k & 3));
    *raw = (int32_t)h[0]; *stored = (int32_t)h[1];
    if (*stored > n - WRAP_HEADER || *stored < 0 || *raw < 0) return WRAP_E_FORMAT;     // :582-583
    return *stored >= *raw ? *stored : *raw;                                            // :587-596
}

// Prep: returns the packet's size or its status (cap: the output capacity; INT32_MAX = no limit, the packed unwrap) and
// writes its decode entry.  A compressed packet decodes its stored bytes into exactly raw bytes (dec_cap = raw >= 1); a
// stored or rejected packet gets the neutral entry (0, 0).
SIMT_DEV int32_t unwrap_prep_one(const uint8_t* p, int32_t n, int32_t cap, int32_t* dec_len, int32_t* dec_cap)
{
    int32_t raw = 0, stored = 0;
    int32_t size = unwrap_header(p, n, &raw, &stored);
    if (size >= 0 && size > cap) size = WRAP_E_ARG;                                     // a slot too small
    const bool comp = size >= 0 && stored < raw;
    *dec_len = comp ? stored : 0;
    *dec_cap = comp ? raw : 0;
    return size;
}

// Finish, called by all 32 lanes of a warp with the same arguments: size = what the prep returned, (dec_len, dec_cap) its
// decode entry, read = the decoder's result for it.  Copies a stored payload to dst and returns out_len: the stored
// length, bytes restored when the decoder read exactly the stored bytes (LZ4Codec.cs:595), else LZ4B200_E_FORMAT; a
// rejected packet keeps its status.
SIMT_DEV int32_t unwrap_finish_one(const uint8_t* p, int32_t size, int32_t dec_len, int32_t dec_cap, int32_t read, uint8_t* dst, int lane)
{
    if (size < 0) return size;
    if (dec_cap > 0) return read == dec_len ? dec_cap : WRAP_E_FORMAT;
    if (size > 0) {
        const InputSrc s{p + WRAP_HEADER};
        group_copy<32, false>(dst, s, (uint32_t)size, lane, 0xFFFFFFFFu);
    }
    return size;
}

}  // namespace lz4b200
