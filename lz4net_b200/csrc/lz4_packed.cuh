// lz4_packed.cuh -- where the blocks of a packed unknown-size decode land (capi.cu lz4b200_decode_batch_packed,
// lz4b200_unwrap_batch_packed, lz4b200_decode_batch_packed_to_device).
//
// The blocks have been measured (size[i], negative = malformed) and their sizes scanned (off[0..n]: the exclusive prefix
// sum of max(size, 0), off[n] the total).  The placement step between the scan and the decode gives block i the capacity
// max(size[i], 0) -- a malformed block gets 0, and the decoder rejects it without writing a byte -- and decides whether the
// decoders run at all: `fits`, the gate they read.
//
// A batch decoded in one piece starts at 0 (base = 0, no absolute offsets: the scan's are final).  A batch that comes
// through the host pipeline is decoded a stage at a time, and a stage's blocks start where the earlier stages' end: base =
// the running total the previous stage left, abs_off[i] = base + off[i], and the stage leaves base + off[n] for the next.
// A stage fits when everything up to its end fits; the running total never shrinks, so no stage behind one that does not
// fit fits, and nothing is ever written behind total_cap.
#pragma once
#include "simt.cuh"

namespace lz4b200 {

// Thread i of at least max(n, 1).  abs_off and total may be null (the batch in one piece).
SIMT_DEV void packed_place(int64_t i, const int32_t* size, const int64_t* off, int32_t n, int64_t base, int64_t total_cap,
                           int32_t* cap, int64_t* abs_off, int* fits, int64_t* total)
{
    if (i < n) {
        cap[i] = size[i] > 0 ? size[i] : 0;
        if (abs_off) abs_off[i] = base + off[i];
    }
    if (i == 0) {
        const int64_t end = base + off[n];
        *fits = end <= total_cap;
        if (total) *total = end;
    }
}

}  // namespace lz4b200
