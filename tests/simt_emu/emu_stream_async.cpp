// TEST INFRASTRUCTURE ONLY: the per-thread rules of the asynchronous LZ4Stream calls (lz4net_b200/csrc/lz4_stream.cuh
// stream_cut_one, stream_chunk_failed) compiled in emulation mode (see simt_emu.h) and exposed to
// tests/test_stream_async_emu.py through a C interface.  Not part of the product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_stream.cuh"

using namespace lz4b200;

namespace {

// The kernels' threads on one warp: the lanes take entries with a stride of 32 and meet after every round, so the
// scheduler interleaves them in its seeded order.
struct CutJob { int64_t first; int32_t m, block_size; int64_t n; int64_t* so; int32_t* len; int64_t* dof; int32_t* cap; };
void cut_entry(int lane, void* arg)
{
    CutJob* j = (CutJob*)arg;
    for (int64_t i0 = 0; i0 < j->m; i0 += 32) {
        if (i0 + lane < j->m) stream_cut_one(i0 + lane, j->first, j->block_size, j->n, j->so, j->len, j->dof, j->cap);
        simt::syncwarp(0xFFFFFFFFu);
    }
}

struct StatusJob { const int32_t* comp_len; const int32_t* stored; const int32_t* res; int32_t m; int* failed; };
void status_entry(int lane, void* arg)
{
    StatusJob* j = (StatusJob*)arg;
    for (int64_t i0 = 0; i0 < j->m; i0 += 32) {
        const int64_t i = i0 + lane;
        if (i < j->m && stream_chunk_failed(j->stored[i], j->comp_len[i], j->res[i])) *j->failed = 1;
        simt::syncwarp(0xFFFFFFFFu);
    }
}

}  // namespace

extern "C" {

// lz4_stream_cut_kernel: the chunk table of a stage of m chunks from chunk `first` of a stream of n bytes
void emu_stream_cut(int64_t first, int32_t m, int32_t block_size, int64_t n, int64_t* so, int32_t* len, int64_t* dof, int32_t* cap,
                    uint64_t sched_seed)
{
    CutJob j{first, m, block_size, n, so, len, dof, cap};
    simt_emu::run_warp(cut_entry, &j, sched_seed);
}

// lz4_stream_status_kernel over the stages of one call, in order, each over its m[k] entries (arrays back to back), onto
// one failure flag that the call clears first; returns the flag
int emu_stream_status(int32_t stages, const int32_t* m, const int32_t* comp_len, const int32_t* stored, const int32_t* res,
                      uint64_t sched_seed)
{
    int failed = 0;
    int64_t at = 0;
    for (int32_t k = 0; k < stages; k++) {
        StatusJob j{comp_len + at, stored + at, res + at, m[k], &failed};
        simt_emu::run_warp(status_entry, &j, sched_seed + (uint64_t)k);
        at += m[k];
    }
    return failed;
}

}
