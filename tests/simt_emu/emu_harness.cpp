// TEST INFRASTRUCTURE ONLY: compiles the kernel headers of lz4net_b200/csrc in emulation mode (see simt_emu.h) and
// exposes them to the CPU-side pytest suite through a C interface.  Not part of the product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_decode.cuh"
#include "lz4_decode_lpb.cuh"
#include "lz4_encode.cuh"
#include "lz4hc_encode.cuh"
#include "lz4hc_warp.cuh"
#include "lz4hc_window.cuh"
#include "lz4_measure.cuh"
#include <stdlib.h>
#include <vector>

using namespace lz4b200;

namespace {

struct DecJob {
    int G; bool known; int nblocks;
    const uint8_t* const* src; const int* isize; uint8_t* const* dst; const int* cap; int* result;
    bool staged;
    DecRing<32> r32[1]; DecRing<16> r16[2]; DecRing<8> r8[4]; DecRing<4> r4[8];
    DecStage<32> s32[1]; DecStage<16> s16[2]; DecStage<8> s8[4]; DecStage<4> s4[8];
    template <int G> DecStage<G>* stages();
    template <int G> DecRing<G>* rings();
};
template <> DecRing<32>* DecJob::rings<32>() { return r32; }
template <> DecRing<16>* DecJob::rings<16>() { return r16; }
template <> DecRing<8>*  DecJob::rings<8>()  { return r8; }
template <> DecRing<4>*  DecJob::rings<4>()  { return r4; }
template <> DecStage<32>* DecJob::stages<32>() { return s32; }
template <> DecStage<16>* DecJob::stages<16>() { return s16; }
template <> DecStage<8>*  DecJob::stages<8>()  { return s8; }
template <> DecStage<4>*  DecJob::stages<4>()  { return s4; }

template <int G, bool KNOWN>
void dec_lane(int wl, DecJob* j)
{
    const int leader = wl & ~(G - 1);
    const int grp = wl / G;
    const uint32_t gmask = (G == 32) ? 0xFFFFFFFFu : (((1u << G) - 1u) << leader);
    DecStream<G> st;
    st.ring = &j->rings<G>()[grp]; st.lane = wl - leader; st.gmask = gmask;
    st.gbase = 0;
    // every group walks the block list with a stride, like the kernel's dynamic hand-out
    for (int b = grp; b < j->nblocks; b += 32 / G) {
        int r = j->staged ? decode_block_staged<G, KNOWN>(st, &j->stages<G>()[grp], j->src[b], j->isize[b], j->dst[b], j->cap[b])
                          : decode_block<G, KNOWN>(st, j->src[b], j->isize[b], j->dst[b], j->cap[b]);
        if (st.lane == 0) j->result[b] = r;
    }
}

void dec_entry(int lane, void* arg)
{
    DecJob* j = (DecJob*)arg;
    switch (j->G) {
    case 4:  j->known ? dec_lane<4, true>(lane, j)  : dec_lane<4, false>(lane, j); break;
    case 8:  j->known ? dec_lane<8, true>(lane, j)  : dec_lane<8, false>(lane, j); break;
    case 16: j->known ? dec_lane<16, true>(lane, j) : dec_lane<16, false>(lane, j); break;
    default: j->known ? dec_lane<32, true>(lane, j) : dec_lane<32, false>(lane, j); break;
    }
}

// lane-per-block decoder: the whole warp loop of the kernel, blocks handed out through the counter
struct LpbJob { LpbBatch a; uint32_t counter; int known; int geo; void* sh; };
void lpb_entry(int lane, void* arg)
{
    LpbJob* j = (LpbJob*)arg;
    // geo 0: the kernel's geometry; geo 1: larger rings, 64-byte runs, requests one iteration ahead, one sequence per iteration
    // (every template path of the header stays compiled and tested)
    if (j->geo == 1) {
        typedef LpbGeom<256, 512, 64, 1, 1> G;
        j->known ? lpb_decode_warp<true, G>((LpbShared<G>*)j->sh, j->a, &j->counter, lane) : lpb_decode_warp<false, G>((LpbShared<G>*)j->sh, j->a, &j->counter, lane);
    } else {
        typedef LpbGeom<128, 256, 32, 0, 2> G;
        j->known ? lpb_decode_warp<true, G>((LpbShared<G>*)j->sh, j->a, &j->counter, lane) : lpb_decode_warp<false, G>((LpbShared<G>*)j->sh, j->a, &j->counter, lane);
    }
}

struct EncJob {
    int variant; EncTune tune;
    int nblocks; const uint8_t* const* src; const int* n; uint8_t* const* dst; const int* cap; int* result;
    EncShared* sh;
};

void enc_entry(int lane, void* arg)
{
    EncJob* j = (EncJob*)arg;
    for (int b = 0; b < j->nblocks; b++) {
        int r = j->variant == 1 ? encode_block<1>(j->sh, j->src[b], j->n[b], j->dst[b], j->cap[b], lane, j->tune)
                                : encode_block<2>(j->sh, j->src[b], j->n[b], j->dst[b], j->cap[b], lane, j->tune);
        if (lane == 0) j->result[b] = r;
    }
}

// measure pass: one lane per block like the kernel; the lanes take blocks with a stride and meet after every round of
// 32 blocks, so the scheduler interleaves them in its seeded order
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

void emu_decode(int G, int known, int nblocks, const uint8_t* const* src, const int* isize,
                uint8_t* const* dst, const int* cap, int* result, uint64_t sched_seed)
{
    DecJob* j = new DecJob();
    j->staged = G >= 100; G %= 100;
    j->G = G; j->known = known != 0; j->nblocks = nblocks; j->src = src; j->isize = isize; j->dst = dst; j->cap = cap; j->result = result;
    simt_emu::run_warp(dec_entry, j, sched_seed);
    delete j;
}

void emu_decode_lpb(int geo, int known, int nblocks, const uint8_t* const* src, const int* isize,
                    uint8_t* const* dst, const int* cap, int* result, uint64_t sched_seed)
{
    std::vector<int64_t> so(nblocks), dof(nblocks);
    const uint8_t* sb = nblocks ? src[0] : nullptr; uint8_t* db = nblocks ? dst[0] : nullptr;
    for (int i = 0; i < nblocks; i++) { so[i] = src[i] - sb; dof[i] = dst[i] - db; }
    LpbJob j;
    j.a = LpbBatch{sb, so.data(), isize, db, dof.data(), cap, result, nblocks};
    j.counter = 0; j.known = known; j.geo = geo;
    j.sh = aligned_alloc(128, sizeof(LpbShared<LpbGeom<256, 512>>));
    memset(j.sh, 0xA5, sizeof(LpbShared<LpbGeom<256, 512>>));
    simt_emu::run_warp(lpb_entry, &j, sched_seed);
    free(j.sh);
}

// the HC encoder is one thread per block: plain scalar code, no warp needed
int emu_encode_hc(const uint8_t* src, int n, uint8_t* dst, int cap)
{
    void* st = aligned_alloc(16, HC_STATE_BYTES);
    memset(st, 0x5A, HC_STATE_BYTES);               // stale garbage, like a reused arena slot
    int r = hc_encode_block(st, src, n, dst, cap);
    free(st);
    return r;
}

// the warp-per-block HC encoder (static index); returns HCW_FALLBACK when the block is handed to the scalar kernel
struct HcwJob { const uint8_t* src; int n; uint8_t* dst; int cap; int result; void* sm; void* index; int smem; };
static void hcw_entry(int lane, void* arg)
{
    HcwJob* j = (HcwJob*)arg;
    const int r = j->smem ? hcw_encode_block<true>(simt::smem_ref_of(j->sm), j->index, j->src, j->n, j->dst, j->cap, lane)
                          : hcw_encode_block<false>(simt::smem_ref_of(j->sm), j->index, j->src, j->n, j->dst, j->cap, lane);
    if (lane == 0) j->result = r;
}
int emu_encode_hcw(const uint8_t* src, int n, uint8_t* dst, int cap, uint64_t sched_seed, int smem)
{
    HcwJob j{src, n, dst, cap, 0, aligned_alloc(16, HCW_SMEM_BYTES), aligned_alloc(16, HCW_INDEX_BYTES), smem};
    memset(j.sm, 0x5A, HCW_SMEM_BYTES); memset(j.index, 0xA5, HCW_INDEX_BYTES);     // stale garbage, like a reused slot
    simt_emu::run_warp(hcw_entry, &j, sched_seed);
    free(j.sm); free(j.index);
    return j.result;
}

// the warp-per-block HC encoder over a sliding 64 KiB window (blocks above 64 KiB); returns the bytes written, 0 (did not
// fit) or HCW_FALLBACK (handed back to the thread-per-block kernel)
struct WinJob { const uint8_t* src; int n; uint8_t* dst; int cap; int result; void* index; };
static void win_entry(int lane, void* arg)
{
    WinJob* j = (WinJob*)arg;
    const int r = hcww_encode_block(j->index, j->src, j->n, j->dst, j->cap, lane);
    if (lane == 0) j->result = r;
}
int emu_encode_hcw_window(const uint8_t* src, int n, uint8_t* dst, int cap, uint64_t sched_seed)
{
    WinJob j{src, n, dst, cap, 0, aligned_alloc(16, HCWW_INDEX_BYTES)};
    memset(j.index, 0xA5, HCWW_INDEX_BYTES);                          // stale garbage, like a reused arena slot
    simt_emu::run_warp(win_entry, &j, sched_seed);
    free(j.index);
    return j.result;
}

// variant: how the round finds same-hash lanes (1 always exact votes, 2 optimistic); the last three are EncTune's fields
void emu_encode(int variant, int lane_copy_max, int probe_max, int wide_min, int nblocks, const uint8_t* const* src,
                const int* n, uint8_t* const* dst, const int* cap, int* result, uint64_t sched_seed)
{
    EncTune tune;
    tune.lane_copy_max = lane_copy_max; tune.probe_max = probe_max; tune.wide_min = wide_min;
    EncJob j{variant, tune, nblocks, src, n, dst, cap, result, (EncShared*)aligned_alloc(16, sizeof(EncShared))};
    simt_emu::run_warp(enc_entry, &j, sched_seed);
    free(j.sh);
}

// cap may be null: INT32_MAX for every block (the unknown-size mode's "no limit")
void emu_measure(int known, int nblocks, const uint8_t* const* src, const int* isize, const int* cap, int* result, uint64_t sched_seed)
{
    MeasureJob j{known, nblocks, src, isize, cap, result};
    simt_emu::run_warp(measure_entry, &j, sched_seed);
}

}
