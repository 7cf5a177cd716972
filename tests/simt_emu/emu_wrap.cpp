// TEST INFRASTRUCTURE ONLY: the Wrap / Unwrap packet steps of lz4net_b200/csrc/lz4_wrap.cuh compiled in emulation mode
// (see simt_emu.h) and exposed to tests/test_wrap_device_emu.py through a C interface.  Not part of the product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_wrap.cuh"

using namespace lz4b200;

namespace {

// the unwrap prep one lane per packet like its kernel; the two finish steps one packet per warp, in order
struct WrapJob {
    int nblocks; const uint8_t* const* src; const int* len; const int* cap; const int* r; uint8_t* const* dst;
    int* out; int* dec_len; int* dec_cap;
};
void unwrap_prep_entry(int lane, void* arg)
{
    WrapJob* j = (WrapJob*)arg;
    for (int b0 = 0; b0 < j->nblocks; b0 += 32) {
        const int b = b0 + lane;
        if (b < j->nblocks) j->out[b] = unwrap_prep_one(j->src[b], j->len[b], j->cap ? j->cap[b] : 0x7FFFFFFF, j->dec_len + b, j->dec_cap + b);
        simt::syncwarp(0xFFFFFFFFu);
    }
}
void wrap_finish_entry(int lane, void* arg)
{
    WrapJob* j = (WrapJob*)arg;
    for (int b = 0; b < j->nblocks; b++) {
        const int r = wrap_finish_one(j->src[b], j->len[b], j->cap[b], j->r[b], j->dst[b], lane);
        if (lane == 0) j->out[b] = r;
    }
}
void unwrap_finish_entry(int lane, void* arg)
{
    WrapJob* j = (WrapJob*)arg;
    for (int b = 0; b < j->nblocks; b++) {
        const int r = unwrap_finish_one(j->src[b], j->len[b], j->dec_len[b], j->dec_cap[b], j->r[b], j->dst[b], lane);
        simt::syncwarp(0xFFFFFFFFu);
        if (lane == 0) j->out[b] = r;
    }
}

}  // namespace

extern "C" {

// unwrap prep: size[i] = the packet's size or status (cap may be null: no limit), (dec_len, dec_cap) its decode entry
void emu_unwrap_prep(int nblocks, const uint8_t* const* src, const int* len, const int* cap, int* size, int* dec_len, int* dec_cap,
                     uint64_t sched_seed)
{
    WrapJob j{nblocks, src, len, cap, nullptr, nullptr, size, dec_len, dec_cap};
    simt_emu::run_warp(unwrap_prep_entry, &j, sched_seed);
}

// wrap finish: packet i from input src[i] (len[i] bytes), capacity cap[i], encoder result r[i], written at dst[i]
void emu_wrap_finish(int nblocks, const uint8_t* const* src, const int* len, const int* cap, const int* r, uint8_t* const* dst,
                     int* out, uint64_t sched_seed)
{
    WrapJob j{nblocks, src, len, cap, r, dst, out, nullptr, nullptr};
    simt_emu::run_warp(wrap_finish_entry, &j, sched_seed);
}

// unwrap finish: packet src[i] with prep size size[i], decode entry (dec_len, dec_cap), decoder result read[i], output dst[i]
void emu_unwrap_finish(int nblocks, const uint8_t* const* src, const int* size, const int* dec_len, const int* dec_cap,
                       const int* read, uint8_t* const* dst, int* out, uint64_t sched_seed)
{
    WrapJob j{nblocks, src, size, nullptr, read, dst, out, (int*)dec_len, (int*)dec_cap};
    simt_emu::run_warp(unwrap_finish_entry, &j, sched_seed);
}

}
