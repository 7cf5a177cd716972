// TEST INFRASTRUCTURE ONLY: the landing step of the asynchronous packed encode (lz4net_b200/csrc/lz4_land.cuh) compiled in
// emulation mode (see simt_emu.h) and exposed to tests/test_land_host_emu.py through a C interface.  Not part of the
// product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_land.cuh"

using namespace lz4b200;

namespace {

// The kernel's loops on one warp: the lanes take entries, then units, with a stride of 32 and meet after every round, so
// the scheduler interleaves them in its seeded order.
struct LandJob {
    const uint8_t* dense; const int64_t* dof; const int32_t* len; const int64_t* off; int32_t m;
    int64_t base, total_cap; uint8_t* dst; int64_t* out_off; int32_t* out_len; int64_t* total_out;
};
void land_entry(int lane, void* arg)
{
    LandJob* j = (LandJob*)arg;
    for (int64_t i0 = 0; i0 <= j->m; i0 += 32) {
        land_place(i0 + lane, j->len, j->off, j->m, j->base, j->out_off, j->out_len, j->total_out);
        simt::syncwarp(0xFFFFFFFFu);
    }
    if (j->base + j->off[j->m] > j->total_cap) return;
    uint8_t* at = j->dst + j->base;
    const int64_t units = land_units(at, j->off[j->m]);
    for (int64_t u0 = 0; u0 < units; u0 += 32) {
        if (u0 + lane < units) land_unit(u0 + lane, j->dense, j->dof, j->off, j->m, at);
        simt::syncwarp(0xFFFFFFFFu);
    }
}

}  // namespace

extern "C" {

// One stage of lz4_land_kernel: base_in (may be null: 0) is read before any lane runs, as the kernel's threads read a
// cell none of them writes.
void emu_land_stage(const uint8_t* dense, const int64_t* dof, const int32_t* len, const int64_t* off, int32_t m,
                    const int64_t* base_in, int64_t total_cap, uint8_t* dst, int64_t* out_off, int32_t* out_len,
                    int64_t* total_out, uint64_t sched_seed)
{
    LandJob j{dense, dof, len, off, m, base_in ? *base_in : 0, total_cap, dst, out_off, out_len, total_out};
    simt_emu::run_warp(land_entry, &j, sched_seed);
}

}
