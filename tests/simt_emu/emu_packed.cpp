// TEST INFRASTRUCTURE ONLY: the placement step of the packed decodes (lz4net_b200/csrc/lz4_packed.cuh) compiled in
// emulation mode (see simt_emu.h) and exposed to tests/test_packed_carry_emu.py through a C interface.  Not part of the
// product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_packed.cuh"

using namespace lz4b200;

namespace {

// one lane per block like the kernel, 32 at a time, at least one round (a stage without blocks still sets its flag)
struct PlaceJob {
    const int32_t* size; const int64_t* off; int32_t n; int64_t base, total_cap;
    int32_t* cap; int64_t* abs_off; int* fits; int64_t* total;
    int32_t room;
};
void place_entry(int lane, void* arg)
{
    PlaceJob* j = (PlaceJob*)arg;
    for (int64_t i0 = 0; i0 == 0 || i0 < j->n; i0 += 32) {
        packed_place(i0 + lane, j->size, j->off, j->n, j->base, j->total_cap, j->cap, j->abs_off, j->fits, j->total, j->room);
        simt::syncwarp(0xFFFFFFFFu);
    }
}

}  // namespace

extern "C" {

// The step of lz4_packed_prep_kernel: base_in (may be null: 0) is read before any lane runs, as the kernel's threads read a
// cell none of them writes; abs_off and total_out may be null.
void emu_packed_place(const int32_t* size, const int64_t* off, int32_t n, const int64_t* base_in, int64_t total_cap, int32_t* cap,
                      int64_t* abs_off, int* fits, int64_t* total_out, uint64_t sched_seed)
{
    PlaceJob j{size, off, n, base_in ? *base_in : 0, total_cap, cap, abs_off, fits, total_out, 0};
    simt_emu::run_warp(place_entry, &j, sched_seed);
}

// The same with `room` bytes of capacity beyond each block's size (the unknown-size packed decodes pass
// PACKED_ROOM_UNKNOWN).
void emu_packed_place_room(const int32_t* size, const int64_t* off, int32_t n, const int64_t* base_in, int64_t total_cap,
                           int32_t* cap, int64_t* abs_off, int* fits, int64_t* total_out, int32_t room, uint64_t sched_seed)
{
    PlaceJob j{size, off, n, base_in ? *base_in : 0, total_cap, cap, abs_off, fits, total_out, room};
    simt_emu::run_warp(place_entry, &j, sched_seed);
}

}
