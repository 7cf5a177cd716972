// TEST INFRASTRUCTURE ONLY: compiles the windowed LZ4HC warp encoder (lz4net_b200/csrc/lz4hc_window.cuh) in emulation mode
// (see simt_emu.h) and exposes it to the CPU-side pytest suite through a C interface (tests/emu_hcw_window.py).  Not part
// of the product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4hc_window.cuh"

#include <stdlib.h>

using namespace lz4b200;

namespace {

struct WinJob { const uint8_t* src; int n; uint8_t* dst; int cap; int result; void* index; };

void win_entry(int lane, void* arg)
{
    WinJob* j = (WinJob*)arg;
    const int r = hcww_encode_block(j->index, j->src, j->n, j->dst, j->cap, lane);
    if (lane == 0) j->result = r;
}

}  // namespace

extern "C" {

size_t emu_hcw_window_index_bytes() { return HCWW_INDEX_BYTES; }

// returns the bytes written, 0 (did not fit) or HCW_FALLBACK (handed back to the thread-per-block kernel)
int emu_encode_hcw_window(const uint8_t* src, int n, uint8_t* dst, int cap, uint64_t sched_seed)
{
    WinJob j{src, n, dst, cap, 0, aligned_alloc(16, HCWW_INDEX_BYTES)};
    memset(j.index, 0xA5, HCWW_INDEX_BYTES);                          // stale garbage, like a reused arena slot
    simt_emu::run_warp(win_entry, &j, sched_seed);
    free(j.index);
    return j.result;
}

}
