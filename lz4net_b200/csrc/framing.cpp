// framing.cpp -- host-side framing on top of the batch ABI: the LZ4Stream chunk format and the Wrap/Unwrap packet.
//
// LZ4Stream (src/LZ4/LZ4Stream.cs) is the reference's block dispatcher: it buffers one block, calls
// LZ4Codec.Encode/EncodeHC with capacity == block length, and writes  varint(flags) varint(rawLen) [varint(compLen)]
// payload  per chunk (FlushCurrentChunk :239-269; reader AcquireNextChunk :274-312; varints :167-187,225-236).
// Here the same byte stream is produced / consumed with ONE batched GPU call for all chunks of a buffer.
// Pure host code: no kernels, no codec arithmetic -- that all lives behind lz4b200_{encode,decode}_batch.
#include "../../include/lz4b200.h"
#include "framing.h"

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

enum : uint64_t { FLAG_COMPRESSED = 1, FLAG_HC = 2 };          // ChunkFlags, LZ4Stream.cs:43-58

inline int varint_size(uint64_t v) { int n = 1; while (v >>= 7) n++; return n; }

inline uint8_t* put_varint(uint8_t* p, uint64_t v)             // LZ4Stream.cs:225-236
{
    for (;;) {
        uint8_t b = (uint8_t)(v & 0x7F);
        v >>= 7;
        *p++ = (uint8_t)(b | (v ? 0x80 : 0));
        if (!v) return p;
    }
}

// LZ4Stream.cs:167-187.  Returns 1 = value read, 0 = clean end of data before the first byte, -1 = truncated.
inline int get_varint(const uint8_t* s, int64_t n, int64_t* pos, uint64_t* out)
{
    uint64_t r = 0; int count = 0;
    for (;;) {
        if (*pos >= n) return count == 0 ? 0 : -1;
        uint8_t b = s[(*pos)++];
        r += (uint64_t)(b & 0x7F) << count;
        count += 7;
        if (!(b & 0x80) || count >= 64) break;
    }
    *out = r;
    return 1;
}

inline uint32_t get_u32le(const uint8_t* p) { return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24; }
inline void put_u32le(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }

}  // namespace

int lz4b200::read_header(const uint8_t* s, int32_t n, int32_t* raw, int32_t* stored)
{
    if (!s || n < 8) return LZ4B200_E_FORMAT;                                            // :577-578
    *raw = (int32_t)get_u32le(s); *stored = (int32_t)get_u32le(s + 4);
    if (*stored > n - 8 || *stored < 0 || *raw < 0) return LZ4B200_E_FORMAT;             // :582-583
    return *stored >= *raw ? *stored : *raw;                                             // :587-596
}

int64_t lz4b200::stream_walk(const uint8_t* s, int64_t n, std::vector<StreamChunk>* out)
{
    int64_t pos = 0, total = 0;
    for (;;) {
        uint64_t flags, raw, clen;
        int r = get_varint(s, n, &pos, &flags);
        if (r == 0) return total;                               // legitimate end (LZ4Stream.cs:281)
        if (r < 0) return LZ4B200_E_FORMAT;
        if (get_varint(s, n, &pos, &raw) != 1) return LZ4B200_E_FORMAT;
        const bool comp = (flags & FLAG_COMPRESSED) != 0;
        clen = raw;
        if (comp && get_varint(s, n, &pos, &clen) != 1) return LZ4B200_E_FORMAT;
        const int32_t rawi = (int32_t)raw, cleni = (int32_t)clen;             // the reference casts to int (:286-287)
        if (rawi < 0 || cleni < 0 || cleni > rawi) return LZ4B200_E_FORMAT;   // :288 corrupted
        if (pos + cleni > n) return LZ4B200_E_FORMAT;                         // :293 short read
        if (comp && (flags >> 2) != 0) return LZ4B200_E_FORMAT;               // :301-303 multi-pass chunks unsupported
        if (out) out->push_back(StreamChunk{pos, rawi, cleni, comp});
        pos += cleni; total += rawi;
    }
}

extern "C" {

int64_t lz4b200_stream_bound(int64_t n, int32_t block_size)
{
    if (n < 0 || block_size < 1) return LZ4B200_E_ARG;
    const int64_t chunks = (n + block_size - 1) / block_size;
    return n + chunks * (1 + 2 * varint_size((uint64_t)block_size));
}

int64_t lz4b200_stream_encode(lz4b200_ctx* ctx, const void* src, int64_t n, int32_t block_size, int hc, void* dst, int64_t dst_cap)
{
    if (!ctx || n < 0 || block_size < 1 || (n > 0 && (!src || !dst))) return LZ4B200_E_ARG;
    if (dst_cap < lz4b200_stream_bound(n, block_size)) return LZ4B200_E_ARG;
    const uint8_t* s = (const uint8_t*)src; uint8_t* d = (uint8_t*)dst;
    const int64_t chunks = (n + block_size - 1) / block_size;
    // groups of chunks bound the temporary slot buffer (capacity == raw length per chunk, LZ4Stream.cs:243-246)
    const int64_t group = std::max<int64_t>(1, (int64_t)(256u << 20) / block_size);
    std::vector<uint8_t> slots;
    std::vector<int64_t> so, dof; std::vector<int32_t> sl, dc, out;
    int64_t w = 0;
    for (int64_t c0 = 0; c0 < chunks; c0 += group) {
        const int64_t c1 = std::min(chunks, c0 + group), m = c1 - c0;
        so.resize(m); dof.resize(m); sl.resize(m); dc.resize(m); out.assign(m, 0);
        const int64_t base = c0 * block_size;
        for (int64_t i = 0; i < m; i++) {
            const int64_t off = (c0 + i) * block_size;
            so[i] = off; dof[i] = off - base;
            sl[i] = dc[i] = (int32_t)std::min<int64_t>(block_size, n - off);
        }
        slots.resize((size_t)(dof[m - 1] + dc[m - 1]));
        int rc = lz4b200_encode_batch(ctx, s, so.data(), sl.data(), slots.data(), dof.data(), dc.data(), out.data(),
                                      (int32_t)m, hc ? LZ4B200_MODE_HC : LZ4B200_MODE_FAST, LZ4B200_MEM_HOST, nullptr);
        if (rc != LZ4B200_OK) return rc;
        for (int64_t i = 0; i < m; i++) {
            const int32_t raw = sl[i], clen = out[i];
            const bool comp = clen > 0 && clen < raw;                         // LZ4Stream.cs:248-255
            uint8_t* p = d + w;
            p = put_varint(p, (comp ? FLAG_COMPRESSED : 0) | (hc ? FLAG_HC : 0));
            p = put_varint(p, (uint64_t)raw);
            if (comp) p = put_varint(p, (uint64_t)clen);
            std::memcpy(p, comp ? slots.data() + dof[i] : s + so[i], (size_t)(comp ? clen : raw));
            w = (p - d) + (comp ? clen : raw);
        }
    }
    return w;
}

int64_t lz4b200_stream_decoded_size(const void* src, int64_t n)
{
    if (n < 0 || (n > 0 && !src)) return LZ4B200_E_ARG;
    return lz4b200::stream_walk((const uint8_t*)src, n, nullptr);
}

int64_t lz4b200_stream_decode(lz4b200_ctx* ctx, const void* src, int64_t n, void* dst, int64_t dst_cap)
{
    if (!ctx || n < 0 || (n > 0 && !src)) return LZ4B200_E_ARG;
    std::vector<lz4b200::StreamChunk> chunks;
    const int64_t total = lz4b200::stream_walk((const uint8_t*)src, n, &chunks);
    if (total < 0) return total;
    if (total > dst_cap || (total > 0 && !dst)) return LZ4B200_E_ARG;
    const uint8_t* s = (const uint8_t*)src; uint8_t* d = (uint8_t*)dst;
    std::vector<int64_t> so, dof; std::vector<int32_t> sl, dc, out;
    int64_t pos = 0;
    for (const lz4b200::StreamChunk& c : chunks) {
        if (!c.compressed) std::memcpy(d + pos, s + c.payload, (size_t)c.raw);           // stored chunk (:295-299)
        else if (c.raw > 0) { so.push_back(c.payload); sl.push_back(c.stored); dof.push_back(pos); dc.push_back(c.raw); }
        pos += c.raw;
    }
    if (!so.empty()) {
        out.assign(so.size(), -1);
        int rc = lz4b200_decode_batch(ctx, s, so.data(), sl.data(), d, dof.data(), dc.data(), out.data(),
                                      (int32_t)so.size(), 1, LZ4B200_MEM_HOST, nullptr);
        if (rc != LZ4B200_OK) return rc;
        // LZ4Codec.Decode(..., knownOutputLength: true) throws unless exactly compLen bytes were consumed
        // (src/LZ4ps/LZ4Codec.Safe.cs:539-542)
        for (size_t i = 0; i < so.size(); i++) if (out[i] != sl[i]) return LZ4B200_E_FORMAT;
    }
    return total;
}

int lz4b200_wrap(lz4b200_ctx* ctx, const void* src, int32_t n, int hc, void* dst, int32_t dst_cap)
{
    // src/LZ4/LZ4Codec.cs:510-543
    if (!ctx || n < 0 || !dst || (n > 0 && !src)) return LZ4B200_E_ARG;
    if ((int64_t)dst_cap < (int64_t)n + 8) return LZ4B200_E_ARG;
    const uint8_t none = 0;                                                              // an empty input is never read
    const int64_t off = 0; int32_t out = 0;
    const int rc = lz4b200_wrap_batch(ctx, src ? src : &none, &off, &n, hc, dst, &off, &dst_cap, &out, 1);
    return rc != LZ4B200_OK ? rc : out;
}

int lz4b200_unwrap_size(const void* src, int32_t n)
{
    int32_t raw, stored;
    return lz4b200::read_header((const uint8_t*)src, n, &raw, &stored);
}

int lz4b200_unwrap(lz4b200_ctx* ctx, const void* src, int32_t n, void* dst, int32_t dst_cap)
{
    const int size = lz4b200_unwrap_size(src, n);
    if (size < 0) return size;
    if (!ctx || size > dst_cap || (size > 0 && !dst)) return LZ4B200_E_ARG;
    uint8_t none;                                                                        // an empty output is never written
    const int64_t off = 0; int32_t out = 0;
    const int rc = lz4b200_unwrap_batch(ctx, src, &off, &n, dst ? dst : &none, &off, &dst_cap, &out, 1);
    return rc != LZ4B200_OK ? rc : out;
}

// ---- batched Wrap / Unwrap (SURVEY.md 8f rank 2): n packets, ONE encode / decode batch ---------------------------------
// Packet i of the batch is exactly what lz4b200_wrap / LZ4Codec.Wrap (src/LZ4/LZ4Codec.cs:510-543) produces for input i:
// u32le rawLen, u32le storedLen, payload (the compressed bytes, or the input itself when compression does not shrink it).
// Inputs: src + src_off[i], src_len[i] bytes.  Packets: dst + dst_off[i], capacity dst_cap[i] >= src_len[i] + 8.
// out_len[i] = packet size (or a negative status for that packet).
int lz4b200_wrap_batch(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len, int high_compression,
                       void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n)
{
    if (!ctx || n < 0) return LZ4B200_E_ARG;
    if (n == 0) return LZ4B200_OK;
    if (!src || !dst || !src_off || !src_len || !dst_off || !dst_cap || !out_len) return LZ4B200_E_ARG;
    const uint8_t* s = (const uint8_t*)src; uint8_t* d = (uint8_t*)dst;
    // the non-empty inputs are encoded, each into its packet's payload with capacity = the input length (:518-523)
    std::vector<int64_t> so, po; std::vector<int32_t> sl, res;
    for (int32_t i = 0; i < n; i++) {
        if (src_len[i] < 0 || (int64_t)dst_cap[i] < (int64_t)src_len[i] + 8) return LZ4B200_E_ARG;
        if (src_len[i] > 0) { so.push_back(src_off[i]); sl.push_back(src_len[i]); po.push_back(dst_off[i] + 8); }
    }
    res.assign(so.size(), 0);
    if (!so.empty()) {
        int rc = lz4b200_encode_batch(ctx, s, so.data(), sl.data(), d, po.data(), sl.data(), res.data(), (int32_t)so.size(),
                                      high_compression ? LZ4B200_MODE_HC : LZ4B200_MODE_FAST, LZ4B200_MEM_HOST, nullptr);
        if (rc != LZ4B200_OK) return rc;
    }
    for (int32_t i = 0, j = 0; i < n; i++) {
        uint8_t* p = d + dst_off[i]; const int32_t len = src_len[i];
        const int32_t r = len > 0 ? res[j++] : 0;
        const int32_t stored = r >= len || r <= 0 ? len : r;      // stored as is unless compression shrinks it
        put_u32le(p, (uint32_t)len); put_u32le(p + 4, (uint32_t)stored);
        if (stored == len) std::memcpy(p + 8, s + src_off[i], (size_t)len);
        out_len[i] = stored + 8;
    }
    return LZ4B200_OK;
}

// Mirror image (src/LZ4/LZ4Codec.cs:574-599).  Packets: src + src_off[i], src_len[i] bytes.  Outputs: dst + dst_off[i],
// capacity dst_cap[i] >= lz4b200_unwrap_size(packet i).  out_len[i] = bytes restored, or LZ4B200_E_FORMAT / E_ARG.
int lz4b200_unwrap_batch(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                         void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n)
{
    if (!ctx || n < 0) return LZ4B200_E_ARG;
    if (n == 0) return LZ4B200_OK;
    if (!src || !dst || !src_off || !src_len || !dst_off || !dst_cap || !out_len) return LZ4B200_E_ARG;
    const uint8_t* s = (const uint8_t*)src; uint8_t* d = (uint8_t*)dst;
    std::vector<int64_t> so, dof; std::vector<int32_t> sl, dc, res, idx;
    for (int32_t i = 0; i < n; i++) {
        const uint8_t* p = s + src_off[i];
        int32_t raw, stored;
        const int size = lz4b200::read_header(p, src_len[i], &raw, &stored);
        if (size < 0) { out_len[i] = size; continue; }
        if (size > dst_cap[i]) { out_len[i] = LZ4B200_E_ARG; continue; }
        if (stored >= raw) { std::memcpy(d + dst_off[i], p + 8, (size_t)stored); out_len[i] = stored; continue; }
        so.push_back(src_off[i] + 8); sl.push_back(stored); dof.push_back(dst_off[i]); dc.push_back(raw); idx.push_back(i);
    }
    if (!so.empty()) {
        res.assign(so.size(), -1);
        int rc = lz4b200_decode_batch(ctx, s, so.data(), sl.data(), d, dof.data(), dc.data(), res.data(), (int32_t)so.size(), 1,
                                      LZ4B200_MEM_HOST, nullptr);
        if (rc != LZ4B200_OK) return rc;
        for (size_t j = 0; j < so.size(); j++) out_len[idx[j]] = res[j] == sl[j] ? dc[j] : LZ4B200_E_FORMAT;
    }
    return LZ4B200_OK;
}

}  // extern "C"
