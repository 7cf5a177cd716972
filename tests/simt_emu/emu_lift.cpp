// TEST INFRASTRUCTURE ONLY: the staging step of the asynchronous decode and Unwrap from device-written offsets
// (lz4net_b200/csrc/lz4_lift.cuh) compiled in emulation mode (see simt_emu.h) and exposed to tests/test_lift_host_emu.py
// through a C interface.  Not part of the product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_lift.cuh"

using namespace lz4b200;

namespace {

// The kernel's loops on one warp: the lanes take entries, then units, with a stride of 32 and meet after every round.
struct LiftJob {
    const uint8_t* src; int64_t src_cap; const int64_t* slot; const int64_t* span; int32_t m; const int32_t* bound;
    int64_t* so; int32_t* sl; int32_t* dc; uint8_t* io; int32_t* out;
};
void lift_entry_fn(int lane, void* arg)
{
    LiftJob* j = (LiftJob*)arg;
    for (int64_t i0 = 0; i0 < j->m; i0 += 32) {
        if (i0 + lane < j->m) lift_entry((int32_t)(i0 + lane), j->src, j->src_cap, j->slot, j->span, j->m, j->bound, j->so, j->sl, j->dc);
        simt::syncwarp(0xFFFFFFFFu);
    }
    const int64_t units = j->slot[j->m] >> 4;
    for (int64_t u0 = 0; u0 < units; u0 += 32) {
        if (u0 + lane < units) lift_unit(u0 + lane, j->src, j->src_cap, j->slot, j->span, j->m, j->bound, j->io);
        simt::syncwarp(0xFFFFFFFFu);
    }
}
void lift_status_fn(int lane, void* arg)
{
    LiftJob* j = (LiftJob*)arg;
    for (int64_t i0 = 0; i0 < j->m; i0 += 32) {
        if (i0 + lane < j->m) lift_status((int32_t)(i0 + lane), j->src_cap, j->span, j->m, j->bound, j->out);
        simt::syncwarp(0xFFFFFFFFu);
    }
}

}  // namespace

extern "C" {

// One stage of lz4_lift_kernel, then (out != null) lz4_lift_status_kernel over out.
void emu_lift_stage(const uint8_t* src, int64_t src_cap, const int64_t* slot, const int64_t* span, int32_t m, const int32_t* bound,
                    int64_t* so, int32_t* sl, int32_t* dc, uint8_t* io, int32_t* out, uint64_t sched_seed)
{
    LiftJob j{src, src_cap, slot, span, m, bound, so, sl, dc, io, out};
    simt_emu::run_warp(lift_entry_fn, &j, sched_seed);
    if (out) simt_emu::run_warp(lift_status_fn, &j, sched_seed + 1);
}

// The slot bytes the host gives a block of `bound` bytes.
int64_t emu_lift_slot_bytes(int32_t bound) { return lift_slot_bytes(bound); }

}
