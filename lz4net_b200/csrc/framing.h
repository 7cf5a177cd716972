// framing.h -- internal interface of framing.cpp, the host-side reader of the framing formats: the LZ4Stream header walk
// and the Wrap packet header, read before any device work by the LZ4Stream decode and the Unwrap calls (capi.cu
// stream_decode, unwrap_packets) and by the size queries of the C ABI.  The writers are on the device (lz4_stream.cuh,
// lz4_wrap.cuh).
#pragma once
#include <stdint.h>

#include <vector>

namespace lz4b200 {

// One chunk of an LZ4Stream: payload at byte `payload` of the stream, `stored` bytes of it (compLen, or rawLen for a
// stored chunk), `raw` bytes decoded.
struct StreamChunk { int64_t payload; int32_t raw; int32_t stored; bool compressed; };

// Walks the chunk headers of a whole stream of n bytes (LZ4Stream.cs:274-312); appends every chunk to *out when out is
// not null.  Returns the total decoded size or LZ4B200_E_FORMAT.
int64_t stream_walk(const uint8_t* s, int64_t n, std::vector<StreamChunk>* out);

// The Wrap packet header (src/LZ4/LZ4Codec.cs:574-599) of a packet of n bytes at s: u32le raw length, u32le stored
// length.  Returns the unwrapped size, or LZ4B200_E_FORMAT for a malformed packet.
int read_header(const uint8_t* s, int32_t n, int32_t* raw, int32_t* stored);

}  // namespace lz4b200
