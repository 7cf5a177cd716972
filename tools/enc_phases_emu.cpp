// enc_phases_emu.cpp -- the fast encoder with its event counters (enc_prof.cuh) on the CPU warp emulator of
// tests/simt_emu, for tools/enc_phases.py: the event counts of a batch without a GPU.  (The emulator has no clock.)
#define LZ4B200_SIMT_EMU 1
#define LZ4B200_ENC_PROF 1
#include "simt_emu.h"
#include "lz4_encode.cuh"
#include <stdlib.h>

using namespace lz4b200;

namespace {
struct Job { const uint8_t* src; int bsize, nblocks; uint8_t* dst; int cap; int* out_len; EncShared* sh; };
void entry(int lane, void* arg)
{
    Job* j = (Job*)arg;
    for (int b = 0; b < j->nblocks; b++) {
        const int r = encode_block<2>(j->sh, j->src + (size_t)b * j->bsize, j->bsize, j->dst + (size_t)b * j->cap, j->cap, lane, EncTune{});
        if (lane == 0) j->out_len[b] = r;
    }
}
}  // namespace

extern "C" void enc_phases_emu_run(const uint8_t* src, int bsize, int nblocks, int* out_len, unsigned long long* rows)
{
    const int cap = bsize + bsize / 255 + 16;
    Job j{src, bsize, nblocks, (uint8_t*)malloc((size_t)nblocks * cap), cap, out_len, (EncShared*)aligned_alloc(16, sizeof(EncShared))};
    for (int k = 0; k < EP_N; k++) enc_prof_emu_row[k] = 0;
    simt_emu::run_warp(entry, &j, 1);
    for (int k = 0; k < EP_N; k++) rows[k] = enc_prof_emu_row[k];
    free(j.dst); free(j.sh);
}
