// TEST INFRASTRUCTURE ONLY: the LZ4Stream frame steps of lz4net_b200/csrc/lz4_stream.cuh compiled in emulation mode
// (see simt_emu.h) and exposed to tests/test_stream_mixed_emu.py through a C interface.  Not part of the product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_stream.cuh"

using namespace lz4b200;

namespace {

// one chunk per warp, in order, like the frame and stored-copy kernels
struct StreamJob {
    int nchunks; const uint8_t* const* src; const int* raw; const uint8_t* const* comp; const int* r; const int* hc;
    uint8_t* const* dst; int* out;
};
void frame_entry(int lane, void* arg)
{
    StreamJob* j = (StreamJob*)arg;
    for (int b = 0; b < j->nchunks; b++) {
        const int32_t w = stream_frame_one(j->src[b], j->raw[b], j->comp[b], j->r[b], j->hc[b] != 0, j->dst[b], lane);
        if (lane == 0) j->out[b] = w;
    }
}
void stored_entry(int lane, void* arg)
{
    StreamJob* j = (StreamJob*)arg;
    for (int b = 0; b < j->nchunks; b++) stream_stored_one(j->src[b], j->raw[b], j->dst[b], lane);
}

}  // namespace

extern "C" {

// frame write: chunk i of raw[i] bytes at src[i], encoder result r[i] with its bytes at comp[i], HC flag hc[i], written at
// dst[i]; out[i] = the frame's size as the frame write returns it, size[i] = stream_frame_size (the frame-size step)
void emu_stream_frame(int nchunks, const uint8_t* const* src, const int* raw, const uint8_t* const* comp, const int* r,
                      const int* hc, uint8_t* const* dst, int* out, int* size, uint64_t sched_seed)
{
    StreamJob j{nchunks, src, raw, comp, r, hc, dst, out};
    simt_emu::run_warp(frame_entry, &j, sched_seed);
    for (int b = 0; b < nchunks; b++) size[b] = stream_frame_size(raw[b], r[b]);
}

// the header alone (lengths too large to copy here): writes header bytes of (raw, r, hc) to out, returns their count
int emu_stream_header(int raw, int r, int hc, uint8_t* out)
{
    const int h = stream_header_size(raw, r);
    for (int k = 0; k < h; k++) out[k] = stream_header_byte(raw, r, hc != 0, k);
    return h;
}

// stored copy: stored[i] bytes of payload[i] to dst[i] (0 = a compressed chunk: nothing)
void emu_stream_stored(int nchunks, const uint8_t* const* payload, const int* stored, uint8_t* const* dst, uint64_t sched_seed)
{
    StreamJob j{nchunks, payload, stored, nullptr, nullptr, nullptr, dst, nullptr};
    simt_emu::run_warp(stored_entry, &j, sched_seed);
}

}
