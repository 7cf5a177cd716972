// framing.cpp -- the host side of the LZ4Stream chunk format and the Wrap / Unwrap packet: it reads headers, it writes none.
//
// LZ4Stream (src/LZ4/LZ4Stream.cs) writes  varint(flags) varint(rawLen) [varint(compLen)] payload  per chunk (reader
// AcquireNextChunk :274-312; varints :167-187).  The host walks those headers (and the 8-byte Wrap packet header) before
// any device work, so that a malformed stream or packet is reported without touching the device, and sizes the outputs
// from them.  The frames and packet headers themselves are written on the device (lz4_stream.cuh, lz4_wrap.cuh) by the
// pipeline in capi.cu, whichever side the caller's bytes are on.  Pure host code: no kernels, no codec arithmetic.
#include "../../include/lz4b200.h"
#include "framing.h"

#include <cstdint>
#include <vector>

namespace {

enum : uint64_t { FLAG_COMPRESSED = 1 };                       // ChunkFlags, LZ4Stream.cs:43-58

inline int varint_size(uint64_t v) { int n = 1; while (v >>= 7) n++; return n; }

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

int64_t lz4b200_stream_decoded_size(const void* src, int64_t n)
{
    if (n < 0 || (n > 0 && !src)) return LZ4B200_E_ARG;
    return lz4b200::stream_walk((const uint8_t*)src, n, nullptr);
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

}  // extern "C"
