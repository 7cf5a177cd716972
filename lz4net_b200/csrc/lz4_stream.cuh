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
// the decode's status, kept on the device (stream_chunk_failed); the decode from a size the device wrote walks the headers
// on the device too (stream_walk_stage).
// This is the library's only writer of the format.
#pragma once
#include "lz4_copy.cuh"
#include "lz4_lift.cuh"

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

// The asynchronous encode (capi.cu run_async, Source::CUT: its stages planned by plan_chunks) holds no per-chunk host
// metadata: each stage's chunk table is computed on the device.  Entry i of the stage whose first chunk is `first`, in a
// stream of n bytes cut into block_size chunks: the chunk is bytes [so, so + len) of the source, encoded into the stage's
// dense slot at dof with capacity cap = len.  Only a stream's last chunk is short, so slot i starts at i * block_size.
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

// ---- the header walk on the device (capi.cu lz4b200_stream_decode_to_device_at_async) --------------------------------
// The decode from a size the device wrote cannot walk the headers on the host: the stream's bytes may still be in flight
// when the call is made.  One warp per stage walks them instead, with exactly the rules of framing.cpp stream_walk, over
// the page-locked source through its device address.  Stage k has `m` chunk slots (the last stage fewer); the walk starts
// from the carry cells the previous stage's walk left (cursor, decoded total, status, S) and writes:
//   - entry i < m of the FRAMED_DECODE sequence for the i-th chunk it walks: so = the payload's offset in the stage's staged
//     span (which the lift keeps at its host alignment mod 16), dof = the output offset, and (sl, dc, stored) = (compLen,
//     rawLen, 0) for a compressed chunk, (0, 0, rawLen) for a stored one.  An empty chunk, and every slot past the last
//     chunk walked, gets the neutral entry (0, 0, -1): the decoders and the stored copy pass over it, the status rule
//     ignores it;
//   - the stage's span [c_k, c_{k+1}) and its lift descriptor (lz4_lift.cuh, one block: slot[0..1], span[0..2], bound);
//   - its carry cells.
// The first event ends the walk for good (later stages only pad): S < 0 or S > src_cap (E_ARG, before any byte is read),
// a malformed header (E_FORMAT), rawLen > block_size, total + rawLen > dst_cap, or a chunk beyond the last stage's slots
// (E_ARG; the last stage parses one more header to tell that from a malformed one).  The header bytes are read by the
// whole warp as a window of 32 aligned 16-byte units, one per lane, reloaded when a header may reach past it; a unit is
// read only when it starts before src + S, so nothing outside the aligned units around [src, src + S) is read.
constexpr int32_t STREAM_WALK_HEADER_MAX = 30;                       // the longest header stream_walk reads: 3 varints of <= 10 bytes
constexpr int32_t STREAM_E_ARG = -1, STREAM_E_FORMAT = -5;           // LZ4B200_E_ARG / LZ4B200_E_FORMAT
constexpr int STREAM_WALK_CELLS = 4;                                 // carry: cursor, decoded total, status, S
constexpr int STREAM_WALK_LIFT_I64 = 5;                              // lift descriptor: int64 slot[2] | span[3], then int32 bound

struct StreamWalkStage {
    const uint8_t* src; int64_t src_cap;
    const int64_t* src_size;                 // the first stage: where S is read (device address); later stages: null
    const int64_t* carry_in;                 // the previous stage's cells (null for the first stage)
    int64_t* carry_out;
    int32_t block_size; int64_t dst_cap;
    int32_t m; bool last;
    int64_t stage_cap;                       // the most bytes the stage's span may hold (its staging buffer, <= INT32_MAX)
    int64_t* so; int64_t* dof; int32_t* sl; int32_t* dc; int32_t* stored;
    int64_t* lift;                           // STREAM_WALK_LIFT_I64 int64, then the int32 bound
};

// The warp's window over the source: lane L holds the aligned unit at base + 16 L (zero when it starts at or past end).
struct StreamWindow { const uint8_t* base; uint4 unit; };

SIMT_DEV void stream_window_load(StreamWindow* win, const uint8_t* at, const uint8_t* end, int lane)
{
    win->base = at - ((uintptr_t)at & 15);
    const uint8_t* u = win->base + 16 * lane;
    win->unit = u < end ? simt::ldg_nc_v4(u) : uint4{0, 0, 0, 0};
}

SIMT_DEV bool stream_window_holds(const StreamWindow& win, const uint8_t* lo, const uint8_t* hi)
{
    return win.base && lo >= win.base && hi <= win.base + 16 * 32;
}

// byte *p (inside the window); called by all 32 lanes with the same p
SIMT_DEV uint32_t stream_window_byte(const StreamWindow& win, const uint8_t* p)
{
    const uint32_t off = (uint32_t)(p - win.base), w = (off >> 2) & 3;
    const uint32_t mine = w == 0 ? win.unit.x : w == 1 ? win.unit.y : w == 2 ? win.unit.z : win.unit.w;
    return (simt::shfl(0xFFFFFFFFu, mine, (int)(off >> 4)) >> (8 * (off & 3))) & 0xFFu;
}

// framing.cpp get_varint over the window: 1 = value read, 0 = clean end before its first byte, -1 = truncated at S.
SIMT_DEV int stream_walk_varint(const StreamWindow& win, const uint8_t* src, int64_t S, int64_t* pos, uint64_t* out)
{
    uint64_t r = 0; int count = 0;
    for (;;) {
        if (*pos >= S) return count == 0 ? 0 : -1;
        const uint32_t b = stream_window_byte(win, src + (*pos)++);
        r += (uint64_t)(b & 0x7F) << count;
        count += 7;
        if (!(b & 0x80) || count >= 64) break;
    }
    *out = r;
    return 1;
}

// One header at *pos (< S), the window holding [*pos, min(*pos + STREAM_WALK_HEADER_MAX, S)).  Returns 0 and the chunk
// (compressed flag, rawLen, compLen or the stored length, and *pos at its payload), or LZ4B200_E_FORMAT.
SIMT_DEV int32_t stream_walk_header(const StreamWindow& win, const uint8_t* src, int64_t S, int64_t* pos, bool* comp, int32_t* raw,
                                    int32_t* clen)
{
    uint64_t flags = 0, r = 0, c = 0;
    if (stream_walk_varint(win, src, S, pos, &flags) != 1) return STREAM_E_FORMAT;
    if (stream_walk_varint(win, src, S, pos, &r) != 1) return STREAM_E_FORMAT;
    *comp = (flags & STREAM_FLAG_COMPRESSED) != 0;
    c = r;
    if (*comp && stream_walk_varint(win, src, S, pos, &c) != 1) return STREAM_E_FORMAT;
    *raw = (int32_t)r; *clen = (int32_t)c;                                  // cast to int as the reference does
    if (*raw < 0 || *clen < 0 || *clen > *raw) return STREAM_E_FORMAT;
    if (*pos + *clen > S) return STREAM_E_FORMAT;
    if (*comp && (flags >> 2) != 0) return STREAM_E_FORMAT;
    return 0;
}

SIMT_DEV void stream_walk_neutral(int32_t i, const StreamWalkStage& w)
{
    w.so[i] = 0; w.dof[i] = 0; w.sl[i] = 0; w.dc[i] = 0; w.stored[i] = -1;
}

// One stage of the walk, called by all 32 lanes of a warp with the same arguments.
SIMT_DEV void stream_walk_stage(const StreamWalkStage& w, int lane)
{
    int64_t cur = 0, total = 0, status = 0, S = 0;
    if (w.carry_in) {
        cur = w.carry_in[0]; total = w.carry_in[1]; status = w.carry_in[2]; S = w.carry_in[3];
    } else {
        S = *w.src_size;
        if (S < 0 || S > w.src_cap) status = STREAM_E_ARG;
    }
    const int64_t c0 = cur;
    const uint8_t* end = w.src + (status ? 0 : S);
    StreamWindow win{nullptr, uint4{0, 0, 0, 0}};
    int32_t i = 0;                                                          // entries written
    while (status == 0 && cur < S && (i < w.m || w.last)) {
        const uint8_t* at = w.src + cur;
        const uint8_t* need = w.src + (S - cur < STREAM_WALK_HEADER_MAX ? S : cur + STREAM_WALK_HEADER_MAX);
        if (!stream_window_holds(win, at, need)) stream_window_load(&win, at, end, lane);
        int64_t pos = cur;
        bool comp = false; int32_t raw = 0, clen = 0;
        const int32_t h = stream_walk_header(win, w.src, S, &pos, &comp, &raw, &clen);
        if (h) { status = h; break; }
        if (i == w.m || raw > w.block_size || total + raw > w.dst_cap || pos + clen - c0 > w.stage_cap) { status = STREAM_E_ARG; break; }
        if (lane == 0) {
            if (raw == 0) {
                stream_walk_neutral(i, w);
            } else {
                w.so[i] = (int64_t)((uintptr_t)(w.src + c0) & 15) + (pos - c0);
                w.dof[i] = total;
                w.sl[i] = comp ? clen : 0; w.dc[i] = comp ? raw : 0; w.stored[i] = comp ? 0 : raw;
            }
        }
        i++; total += raw; cur = pos + clen;
    }
    for (int32_t j = i + lane; j < w.m; j += 32) stream_walk_neutral(j, w);
    if (lane == 0) {
        w.carry_out[0] = cur; w.carry_out[1] = total; w.carry_out[2] = status; w.carry_out[3] = S;
        // the lift's one block: slot [0, slot_bytes(span)), span [c0, cur), src_off[n] = cur (<= S <= src_cap)
        int64_t* slot = w.lift;
        int64_t* span = w.lift + 2;
        slot[0] = 0; slot[1] = lift_slot_bytes((int32_t)(cur - c0));
        span[0] = c0; span[1] = cur; span[2] = cur;
        *(int32_t*)(w.lift + STREAM_WALK_LIFT_I64) = (int32_t)w.stage_cap;
    }
}

// The call's result from the last stage's carry cells and the decode's failure flag: the walk's status (the size check
// first), then a cursor short of S (more chunks than the slots: E_ARG), then a chunk that did not decode (E_FORMAT), else
// the decoded size.
SIMT_DEV int64_t stream_walk_result(const int64_t* carry, int failed)
{
    return carry[2] ? carry[2] : carry[0] != carry[3] ? (int64_t)STREAM_E_ARG : failed ? (int64_t)STREAM_E_FORMAT : carry[1];
}

}  // namespace lz4b200
