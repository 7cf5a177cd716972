// TEST INFRASTRUCTURE ONLY: compiles the measure-pass header (lz4net_b200/csrc/lz4_measure.cuh) in emulation mode (see
// simt_emu.h) and exposes it to the CPU-side pytest suite through a C interface (tests/emu_measure.py).  Not part of the
// product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_measure.cuh"

using namespace lz4b200;

namespace {

// one lane per block like the kernel; the lanes take blocks with a stride and meet after every round of 32 blocks, so the
// scheduler interleaves them in its seeded order
struct MeasureJob { int known, nblocks; const uint8_t* const* src; const int* isize; const int* cap; int* result; };

void measure_entry(int lane, void* arg)
{
    MeasureJob* j = (MeasureJob*)arg;
    for (int b0 = 0; b0 < j->nblocks; b0 += 32) {
        const int b = b0 + lane;
        if (b < j->nblocks) {
            const int cap = j->cap ? j->cap[b] : 0x7FFFFFFF;
            j->result[b] = j->known ? measure_block<true>(j->src[b], j->isize[b], cap) : measure_block<false>(j->src[b], j->isize[b], cap);
        }
        simt::syncwarp(0xFFFFFFFFu);
    }
}

}  // namespace

extern "C" {

// cap may be null: INT32_MAX for every block (the unknown-size mode's "no limit")
void emu_measure(int known, int nblocks, const uint8_t* const* src, const int* isize, const int* cap, int* result, uint64_t sched_seed)
{
    MeasureJob j{known, nblocks, src, isize, cap, result};
    simt_emu::run_warp(measure_entry, &j, sched_seed);
}

}
