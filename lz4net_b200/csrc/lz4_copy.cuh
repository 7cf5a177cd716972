// lz4_copy.cuh -- group-cooperative byte movers shared by the decoder and the encoders.
//
// A "group" is G consecutive lanes of a warp (G = 32, 16 or 8) that own one LZ4 block together.  Every routine is
// called by all lanes of the group with identical (group-uniform) arguments apart from `lane` (0..G-1).
// Sources are either a power-of-two ring in shared memory (the TMA-staged compressed stream) or global memory.
// Destinations are global memory.  Bulk moves are 128-bit: the destination is aligned with a byte-wise head, the
// source is read as two aligned 128-bit words and funnel-shifted into place (SHF), so every global transaction
// is a full, coalesced 16 B * G segment.
#pragma once
#include "simt.cuh"

namespace lz4b200 {

// bytes [r, r+16) of the 32-byte pair (lo, hi); r in 0..15, group-uniform
SIMT_DEV uint4 shift16(uint4 lo, uint4 hi, uint32_t r)
{
    uint32_t w0, w1, w2, w3, w4;
    switch (r >> 2) {
    case 0:  w0 = lo.x; w1 = lo.y; w2 = lo.z; w3 = lo.w; w4 = hi.x; break;
    case 1:  w0 = lo.y; w1 = lo.z; w2 = lo.w; w3 = hi.x; w4 = hi.y; break;
    case 2:  w0 = lo.z; w1 = lo.w; w2 = hi.x; w3 = hi.y; w4 = hi.z; break;
    default: w0 = lo.w; w1 = hi.x; w2 = hi.y; w3 = hi.z; w4 = hi.w; break;
    }
    const uint32_t bs = (r & 3) * 8;
    uint4 o;
    o.x = simt::funnel_r(w0, w1, bs);
    o.y = simt::funnel_r(w1, w2, bs);
    o.z = simt::funnel_r(w2, w3, bs);
    o.w = simt::funnel_r(w3, w4, bs);
    return o;
}

// little-endian 32-bit read at an arbitrary byte position of the (read-only) input
SIMT_DEV uint32_t in32(const uint8_t* src, int p)
{
    const uint8_t* a = (const uint8_t*)((uintptr_t)(src + p) & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)((uintptr_t)(src + p) & 3) * 8;
    const uint32_t lo = simt::ldg_nc_u32(a);
    const uint32_t hi = sh ? simt::ldg_nc_u32(a + 4) : 0u;           // (never touches a word holding no wanted byte)
    return simt::funnel_r(lo, hi, sh);
}

// The same read through a per-block word view of the input: base rounded down to 4 bytes + a 32-bit word index, so the
// address is one IMAD.WIDE instead of a 64-bit add, align and re-add.
struct InWords {
    const uint32_t* w; uint32_t sk; uint64_t keep;
    SIMT_MEM void init(const uint8_t* src) { sk = (uint32_t)((uintptr_t)src & 3); w = (const uint32_t*)(src - sk); keep = simt::l2_policy_keep(); }
    SIMT_MEM uint32_t at(int p) const
    {
        const uint32_t q = (uint32_t)p + sk, i = q >> 2, sh = (q & 3u) * 8u;
        const uint32_t lo = simt::ldg_nc_u32(w + i);
        const uint32_t hi = sh ? simt::ldg_nc_u32(w + i + 1) : 0u;
        return simt::funnel_r(lo, hi, sh);
    }
    // The same read split in two, so that the caller decides where the warp waits for the data: raw() issues the loads
    // (POLICY 0: plain read-only path; 1: the same with an L2 evict-last hint -- the block is probed again at random
    // positions until its parse is over), word() assembles the value.
    struct Raw { uint32_t lo, hi, sh; };
    template <int POLICY>
    SIMT_MEM Raw raw(int p) const
    {
        const uint32_t q = (uint32_t)p + sk, i = q >> 2;
        Raw r; r.sh = (q & 3u) * 8u;
        // Both words unconditionally (no predicate on the critical path).  Callers only pass positions p <= n - 6 (probe
        // positions <= n - 13, match-count positions < n - 5), so word i + 1 always holds the input byte p + 4: no word
        // without an input byte is ever touched (tests/test_kernels_emu.py::test_encode_never_reads_past_the_input).
        if (POLICY == 1) { r.lo = simt::ldg_nc_hint_u32(w + i, keep); r.hi = simt::ldg_nc_hint_u32(w + i + 1, keep); }
        else             { r.lo = simt::ldg_nc_u32(w + i); r.hi = simt::ldg_nc_u32(w + i + 1); }
        return r;
    }
    static SIMT_MEM uint32_t word(const Raw& r) { return simt::funnel_r(r.lo, r.hi, r.sh); }
    // The 4 bytes [p-4, p) (byte p-1 in the top byte), for the backward catch-up.  The caller passes 1 <= p < n: the word
    // holding byte p is read when part of it is wanted, the word before it only when that is not the first word of the
    // block, so no word without an input byte -- and none in front of src -- is ever touched.  Bytes in front of src
    // come back as zeros (tests/test_encode_deferred_catchup.py::test_catchup_never_reads_before_the_input).
    SIMT_MEM uint32_t back(int p) const
    {
        const uint32_t q = (uint32_t)p + sk, i = q >> 2, sh = (q & 3u) * 8u;
        const uint32_t lo = i ? simt::ldg_nc_u32(w + i - 1) : 0u;
        const uint32_t hi = sh ? simt::ldg_nc_u32(w + i) : 0u;
        return simt::funnel_r(lo, hi, sh);
    }
};

// ---- source policies -------------------------------------------------------------------------------------------
// Ring in shared memory: byte i of the source lives at buf[(pos0 + i) & (SIZE-1)].
template <int SIZE>
struct RingSrc {
    static constexpr bool PIPELINED = false;
    const uint8_t* buf; uint32_t pos0;
    SIMT_MEM uint8_t byte(uint32_t i) const { return buf[(pos0 + i) & (SIZE - 1)]; }
    SIMT_MEM uint32_t misalign(uint32_t i) const { return (pos0 + i) & 15; }
    // aligned 16-byte word containing source byte i (lo) and the following word (hi)
    SIMT_MEM uint4 word(uint32_t i, int k) const
    {
        return *(const uint4*)(buf + (((pos0 + i) & ~15u) + 16u * k & (SIZE - 1)));
    }
};
// Global memory written earlier by this same group (decoder back-references): coherent loads.
struct GlobalSrc {
    static constexpr bool PIPELINED = false;
    const uint8_t* p;
    SIMT_MEM uint8_t byte(uint32_t i) const { return simt::ldg_u8(p + i); }
    SIMT_MEM uint32_t misalign(uint32_t i) const { return (uint32_t)((uintptr_t)(p + i) & 15); }
    SIMT_MEM uint4 word(uint32_t i, int k) const
    {
        return simt::ldg_v4((const uint8_t*)(((uintptr_t)(p + i)) & ~(uintptr_t)15) + 16 * k);
    }
};
// Global memory that is a kernel input (encoder literals): read-only path.
struct InputSrc {
    static constexpr bool PIPELINED = true;
    const uint8_t* p;
    SIMT_MEM uint8_t byte(uint32_t i) const { return simt::ldg_nc_u8(p + i); }
    SIMT_MEM uint32_t misalign(uint32_t i) const { return (uint32_t)((uintptr_t)(p + i) & 15); }
    SIMT_MEM uint4 word(uint32_t i, int k) const
    {
        return simt::ldg_nc_v4((const uint8_t*)(((uintptr_t)(p + i)) & ~(uintptr_t)15) + 16 * k);
    }
};

// Copy n bytes src[0..n) -> dst[0..n).  No overlap between the source bytes and the bytes written by this call
// (the caller guarantees it).  When SYNC_EACH is set the source of iteration k may have been written by iteration
// k-1 of this very call (long self-overlapping matches copied at a distance >= one iteration's span), so the group
// is synchronised between iterations.
template <int G, bool SYNC_EACH, class Src>
SIMT_DEV void group_copy(uint8_t* dst, const Src& src, uint32_t n, int lane, uint32_t gmask)
{
    if (n <= (uint32_t)G) {                               // the common short sequence: one predicated byte step
        if ((uint32_t)lane < n) simt::stg_u8(dst + lane, src.byte(lane));
        return;
    }
    if (n < 64) {                                          // a few byte steps
        for (uint32_t i = lane; i < n; i += G) simt::stg_u8(dst + i, src.byte(i));
        return;                                            // (SYNC_EACH sources are >= one iteration span away: no hazard here)
    }
    // head: bring dst to 16-byte alignment (<= 15 bytes)
    const uint32_t head = (uint32_t)(16 - ((uintptr_t)dst & 15)) & 15;
    for (uint32_t i = lane; i < head; i += G) simt::stg_u8(dst + i, src.byte(i));
    if (SYNC_EACH) simt::syncwarp(gmask);
    const uint32_t nvec = (n - head) >> 4;
    const uint32_t r = src.misalign(head);
    uint32_t v0 = 0;
    if (!SYNC_EACH && Src::PIPELINED) {
        // long runs: four vectors per lane per iteration, all loads issued before the first store (one memory round
        // trip per 4 * 16 * G bytes instead of one per 16 * G -- it matters when few warps are resident: the encoders; measured
        // slower for the decoder, whose many warps hide the latency and which pays for the registers in occupancy)
        for (; v0 + 4u * G <= nvec; v0 += 4u * G) {
            uint4 lo[4], hi[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint32_t i = head + ((v0 + k * G + lane) << 4);
                lo[k] = src.word(i, 0);
                if (r) hi[k] = src.word(i, 1);
            }
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint32_t i = head + ((v0 + k * G + lane) << 4);
                simt::stg_v4(dst + i, r ? shift16(lo[k], hi[k], r) : lo[k]);
            }
        }
    }
    for (; v0 < nvec; v0 += G) {
        const uint32_t v = v0 + lane;
        if (v < nvec) {
            const uint32_t i = head + (v << 4);
            uint4 lo = src.word(i, 0), o;
            if (r) { uint4 hi = src.word(i, 1); o = shift16(lo, hi, r); } else o = lo;
            simt::stg_v4(dst + i, o);
        }
        if (SYNC_EACH) simt::syncwarp(gmask);
    }
    const uint32_t done = head + (nvec << 4);
    for (uint32_t i = done + lane; i < n; i += G) simt::stg_u8(dst + i, src.byte(i));
}

// Self-overlapping match (offset < length): dst[i] = dst[i - off] for i in [0,n), i.e. the `off` bytes before dst
// repeated with period `off`.  Written as reads of ONLY those `off` already-final bytes (index i mod off), so no
// intra-call ordering is needed at all (SURVEY.md 7.2-H4: the modular form of original/lz4.c:869-884).
template <int G>
SIMT_DEV void group_copy_periodic(uint8_t* dst, uint32_t off, uint32_t n, int lane)
{
    const uint8_t* base = dst - off;
    uint32_t m = (uint32_t)lane < off ? (uint32_t)lane : (uint32_t)lane % off;
    const uint32_t gm = (uint32_t)G < off ? (uint32_t)G : (uint32_t)G % off;
    for (uint32_t i = lane; i < n; i += G) {
        simt::stg_u8(dst + i, simt::ldg_u8(base + m));
        m += gm; if (m >= off) m -= off;
    }
}

// The decoder's match copy: n bytes from `off` bytes back.
template <int G>
SIMT_DEV void group_copy_match(uint8_t* dst, uint32_t off, uint32_t n, int lane, uint32_t gmask)
{
    constexpr uint32_t SPAN = 16u * G + 16u;              // one 128-bit iteration reads < SPAN bytes ahead of its first source byte
    if (off >= n) {                                        // disjoint
        GlobalSrc s{dst - off};
        group_copy<G, false>(dst, s, n, lane, gmask);
    } else if (n < 4 * SPAN) {
        group_copy_periodic<G>(dst, off, n, lane);
    } else {
        // long run: lay down P bytes (P = a multiple of the period, >= SPAN) with the periodic form, then the rest
        // is an ordinary copy from P bytes back, 128 bits per lane, iteration k reading what iteration k-1 wrote.
        const uint32_t P = off >= SPAN ? off : off * ((SPAN + off - 1) / off);
        if (P != off) group_copy_periodic<G>(dst, off, P, lane);
        else { GlobalSrc s{dst - off}; group_copy<G, false>(dst, s, P, lane, gmask); }
        simt::syncwarp(gmask);
        GlobalSrc s{dst};                                  // == (dst + P) - P
        group_copy<G, true>(dst + P, s, n - P, lane, gmask);
    }
}

}  // namespace lz4b200
