// TEST INFRASTRUCTURE ONLY: the fast encoder (lz4_encode.cuh) with its event counters (enc_prof.cuh) on the CPU warp
// emulator, built with -DLZ4B200_ENC_PROF by tests/emu.py.  One block at a time: its result, its bytes and its event row,
// so that a test can compare the rounds, paths and probes the kernel took with a model of them.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_encode.cuh"
#include <stdlib.h>

using namespace lz4b200;

namespace {
struct Job { int variant; EncTune tune; const uint8_t* src; int n; uint8_t* dst; int cap; int result; EncShared* sh; };
void entry(int lane, void* arg)
{
    Job* j = (Job*)arg;
    const int r = j->variant == 1 ? encode_block<1>(j->sh, j->src, j->n, j->dst, j->cap, lane, j->tune)
                                  : encode_block<2>(j->sh, j->src, j->n, j->dst, j->cap, lane, j->tune);
    if (lane == 0) j->result = r;
}
}  // namespace

// events: the block's counts, in this order: blocks, sequences, rounds, wide rounds, exact rounds, pair rounds, probes
// tried alone, of which hit
extern "C" int emu_encode_events(int variant, int lane_copy_max, int probe_max, int wide_min, const uint8_t* src, int n,
                                 uint8_t* dst, int cap, unsigned long long* events, uint64_t sched_seed)
{
    EncTune tune;
    tune.lane_copy_max = lane_copy_max; tune.probe_max = probe_max; tune.wide_min = wide_min;
    Job j{variant, tune, src, n, dst, cap, 0, (EncShared*)aligned_alloc(16, sizeof(EncShared))};
    for (int k = 0; k < EP_N; k++) enc_prof_emu_row[k] = 0;
    simt_emu::run_warp(entry, &j, sched_seed);
    const int slots[] = {EP_BLOCK, EP_SEQ, EP_ROUND, EP_ROUND_WIDE, EP_EXACT, EP_PAIR, EP_PROBE, EP_PROBE_HIT};
    for (int k = 0; k < (int)(sizeof(slots) / sizeof(slots[0])); k++) events[k] = enc_prof_emu_row[slots[k]];
    free(j.sh);
    return j.result;
}
