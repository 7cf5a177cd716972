// TEST INFRASTRUCTURE ONLY: the device header walk of the LZ4Stream decode from a size the device wrote
// (lz4net_b200/csrc/lz4_stream.cuh stream_walk_stage, stream_walk_result) compiled in emulation mode (see simt_emu.h), next
// to the host walk it restates (lz4net_b200/csrc/framing.cpp stream_walk, compiled in as it is), exposed to
// tests/test_stream_walk_emu.py through a C interface.  Not part of the product.
#define LZ4B200_SIMT_EMU 1
#include "simt_emu.h"
#include "lz4_stream.cuh"
#include "../../lz4net_b200/csrc/framing.cpp"

using namespace lz4b200;

// framing.cpp's single-packet Wrap and Unwrap call the batch ABI, which this unit does not link: never called here.
extern "C" int lz4b200_wrap_batch(lz4b200_ctx*, const void*, const int64_t*, const int32_t*, int, void*, const int64_t*, const int32_t*,
                                  int32_t*, int32_t) { return LZ4B200_E_ARG; }
extern "C" int lz4b200_unwrap_batch(lz4b200_ctx*, const void*, const int64_t*, const int32_t*, void*, const int64_t*, const int32_t*,
                                    int32_t*, int32_t) { return LZ4B200_E_ARG; }

namespace {

void walk_fn(int lane, void* arg) { stream_walk_stage(*(const StreamWalkStage*)arg, lane); }

}  // namespace

extern "C" {

// The walk kernel over `stages` stages of `per` chunk slots (the last one m_last), in order, as run_async chains them: the
// first reads S from *src_size, each later one the previous stage's carry cells.  Stage k's entries go to [k * per, k * per
// + m_k) of so / dof / sl / dc / stored, its lift descriptor (slot[2] | span[3] | bound) to lift + 8 k.  Returns the call's
// result with the decode's failure flag clear (stream_walk_result).
int64_t emu_stream_walk(const uint8_t* src, int64_t src_cap, const int64_t* src_size, int32_t block_size, int64_t dst_cap, int32_t per,
                        int32_t stages, int32_t m_last, int64_t stage_cap, int64_t* so, int64_t* dof, int32_t* sl, int32_t* dc,
                        int32_t* stored, int64_t* lift, uint64_t sched_seed)
{
    int64_t carry[2][STREAM_WALK_CELLS];
    for (int32_t k = 0; k < stages; k++) {
        const int64_t at = (int64_t)k * per;
        const StreamWalkStage w{src, src_cap, k == 0 ? src_size : nullptr, k > 0 ? carry[(k + 1) & 1] : nullptr, carry[k & 1],
                                block_size, dst_cap, k + 1 == stages ? m_last : per, k + 1 == stages, stage_cap,
                                so + at, dof + at, sl + at, dc + at, stored + at, lift + 8 * k};
        simt_emu::run_warp(walk_fn, (void*)&w, sched_seed + (uint64_t)k);
    }
    return stream_walk_result(carry[(stages + 1) & 1], 0);
}

int64_t emu_stream_walk_result(const int64_t* carry, int failed) { return stream_walk_result(carry, failed); }

// framing.cpp stream_walk over n bytes: the total or LZ4B200_E_FORMAT; the chunks it appended before returning (up to cap
// of them) as payload offset, rawLen, stored bytes (compLen, or rawLen) and compressed flag; *count = how many.
int64_t emu_host_walk(const uint8_t* s, int64_t n, int64_t* payload, int32_t* raw, int32_t* len, uint8_t* comp, int64_t cap, int64_t* count)
{
    std::vector<StreamChunk> chunks;
    const int64_t r = stream_walk(s, n, &chunks);
    *count = (int64_t)chunks.size();
    for (size_t i = 0; i < chunks.size() && (int64_t)i < cap; i++) {
        payload[i] = chunks[i].payload; raw[i] = chunks[i].raw; len[i] = chunks[i].stored; comp[i] = chunks[i].compressed;
    }
    return r;
}

int32_t emu_stream_walk_header_max() { return STREAM_WALK_HEADER_MAX; }

}
