// enc_prof.cuh -- opt-in phase attribution for the fast encoder (lz4_encode.cuh).
//
// Off unless LZ4B200_ENC_PROF is defined: every hook is then an empty macro, so the library's kernels are the same
// instructions with or without this header.  tools/enc_phases.py builds its own copies with it defined.
// With it, lane 0 of every warp adds event counts and clock64 cycles per phase to its warp's row of EP_N counters:
//   * device: row (global warp index) of `enc_prof_rows`, a buffer the caller sets; RED.ADD, nothing waits for it;
//   * CPU emulator (tests/simt_emu): one host row, events only (the emulator has no clock).
// A phase's cycles run from one clock read to the next on the warp's own issue stream, so a load's latency is charged to
// the phase that first uses its value, which is where the warp stalls for it.
#pragma once
#include <stdint.h>

namespace lz4b200 {

enum EncProfSlot {
    // events
    EP_BLOCK, EP_SEQ,                       // blocks encoded, sequences parked (with the last literals)
    EP_ROUND, EP_ROUND_WIDE,                // find-match rounds, of which 64 iterations wide
    EP_EXACT,                               // rounds on the exact path
    EP_PAIR,                                // rounds on the pair path: two iterations share a bucket, none more
    EP_PROBE, EP_PROBE_HIT,                 // post-match probes tried alone, of which hit
    EP_FLUSH, EP_LONG_LIT,                  // EMIT calls, literal runs copied by copy_long_literals
    EP_CATCHUP_LONG,                        // catch-ups finished by the whole warp (longer than EMIT's per-lane steps)
    // clock64 cycles
    EP_C_LOADHASH,                          // round: positions, input words, hashes, table reads, candidate loads issued
    EP_C_SAMEHASH,                          // round: same-hash resolution through the table
    EP_C_VOTE,                              // round: candidate words, hit vote, final table writes
    EP_C_EXACT,                             // round: exact path
    EP_C_PROBE,                             // post-match probe alone
    EP_C_CATCHUP,                           // EMIT: backward catch-up of the 32 parked sequences
    EP_C_COUNT,                             // forward match count
    EP_C_PARK,                              // park the record, prefetch, next round's set-up
    EP_C_EMIT,                              // EMIT after the catch-up: prefix sum, limit checks, token / length stores, literal copy
    EP_C_BLOCK,                             // the whole of encode_block_t, table clear included
    EP_N
};

}  // namespace lz4b200

#if defined(LZ4B200_ENC_PROF)
#if defined(LZ4B200_SIMT_EMU)
namespace lz4b200 {
inline uint64_t enc_prof_emu_row[EP_N];
static inline void enc_prof_add(int k, uint64_t v) { if (simt_emu::current_lane() == 0) enc_prof_emu_row[k] += v; }
static inline long long enc_prof_clock() { return 0; }
}
#else
namespace lz4b200 {
static __device__ unsigned long long* enc_prof_rows;
static __device__ __forceinline__ void enc_prof_add(int k, unsigned long long v)
{
    if ((threadIdx.x & 31) == 0) atomicAdd(enc_prof_rows + (size_t)((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * EP_N + k, v);
}
static __device__ __forceinline__ long long enc_prof_clock() { return clock64(); }
}
#endif
#define ENC_PROF_EVENT(k) lz4b200::enc_prof_add((k), 1)
#define ENC_PROF_EVENT_IF(k, c) do { if (c) lz4b200::enc_prof_add((k), 1); } while (0)
#define ENC_PROF_T0(t) long long t = lz4b200::enc_prof_clock()
#define ENC_PROF_LAP(k, t) do { const long long t_ = lz4b200::enc_prof_clock(); lz4b200::enc_prof_add((k), (uint64_t)(t_ - (t))); t = t_; } while (0)
#define ENC_PROF_RESTART(t) do { t = lz4b200::enc_prof_clock(); } while (0)
#else
#define ENC_PROF_EVENT(k) do {} while (0)
#define ENC_PROF_EVENT_IF(k, c) do {} while (0)
#define ENC_PROF_T0(t) do {} while (0)
#define ENC_PROF_LAP(k, t) do {} while (0)
#define ENC_PROF_RESTART(t) do {} while (0)
#endif
