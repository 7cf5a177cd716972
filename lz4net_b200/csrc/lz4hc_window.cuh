// lz4hc_window.cuh -- byte-exact LZ4HC r93 encoder for blocks ABOVE 64 KiB, one warp per block, over a sliding 64 KiB window
// of 64 KiB index segments.
//
// The argument of lz4hc_warp.cuh carries over once r93's window is added.  LZ4HC_Insert (original/lz4hc.c:364-372)
// clamps each chain delta to MAX_DISTANCE = 65535 and stores it at chain[p & 0xFFFF]; both walks stop at ref < ip - 65535
// (:423, :475).  For a search at q with no search at or above q before it, the walk visits
//     the positions of q's hash bucket in [max(1, q - 65535), q), in descending order; then position 0 if q <= 65535
// -- a clamped delta only ever points below the window, and a slot p & 0xFFFF of a position p in the window could only have
// been overwritten by inserting p + 65536 > q, i.e. by a search above q (the kernel hands such a block back, as below).
// The repeat detector (:437-455) still writes only slots of positions below the next search, even when its run is longer
// than 64 KiB and the writes wrap the u16 table, so lz4hc_warp.cuh's hash-collision check still decides for it.
//
// The index is cut into 64 KiB SEGMENTS, segment s holding positions [65536 s, 65536 (s+1)): a stable counting sort per
// segment (`sorted`, positions relative to the segment), each position's place in it (`rank`) and the bucket ends
// (`end`, u32: one bucket may hold all 65536 positions of a segment).  q's window lies in its own segment and the one
// before it, so the candidates of q are
//     sorted_s[rank_s[q]-1], ... down to the start of q's bucket in segment s, then
//     sorted_{s-1}[end_{s-1}[h]-1], ... while in the bucket and >= q - 65535, then position 0 when s = 0.
// Two segments are resident (slot s & 1).  Searches never go down (else the block is handed back), so each segment is
// built at most once, when a search first needs it, and a segment no window covers (a long match jumping over it) is
// never built.  The literal scan stops its 64-position rounds at segment boundaries, so every round and every candidate
// batch stays within the two resident segments.
//
// This header holds the segment layout, its build and the segmented index (HcwwIndex).  The search, the literal scan and
// the parse are lz4hc_warp.cuh's (hcw_search, hcw_scan, hcw_parse), run on HcwwIndex over a HcwBlock<false>.
#pragma once
#include "lz4hc_warp.cuh"

namespace lz4b200 {

constexpr int    HCWW_SEG         = 65536;
// per segment: rank u16[65536] + sorted u16[65536] + end u32[32768]; two segments per warp in flight
constexpr size_t HCWW_SEG_BYTES   = 2u * 65536u * sizeof(uint16_t) + 32768u * sizeof(uint32_t);
constexpr size_t HCWW_INDEX_BYTES = 2u * HCWW_SEG_BYTES;

struct HcwwSeg { uint16_t* rank; uint16_t* sorted; uint32_t* end; };

// ---- the index, one segment --------------------------------------------------------------------------------------------
SIMT_DEV void hcww_build(const HcwBlock<false>& w, const HcwwSeg& g, int s)
{
    const int lane = w.lane, B = s * HCWW_SEG;
    const int lo = B > 1 ? B : 1, hi = B + HCWW_SEG < w.mflimit ? B + HCWW_SEG : w.mflimit;   // positions 1 .. mflimit-1
    const InWords& in = w.in;
    for (uint32_t i = (uint32_t)lane * 4u; i < 32768u; i += 128u) simt::stg_v4(g.end + i, uint4{0, 0, 0, 0});
    simt::syncwarp(HCW_FULL);
    // bucket sizes (u32 counters, global atomics); the hashes are parked in rank[] for the scatter
    for (int base = lo; base < hi; base += 128) {
        InWords::Raw raw[4];
#pragma unroll
        for (int j = 0; j < 4; j++) { const int p = base + 32 * j + lane; if (p < hi) raw[j] = in.raw<0>(p); }     // p <= n - 13
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int p = base + 32 * j + lane;
            if (p < hi) { const uint32_t h = hcw_hash(InWords::word(raw[j])); simt::stg_u16(g.rank + (p - B), h); simt::atomg_add(g.end + h, 1u); }
        }
    }
    simt::syncwarp(HCW_FULL);
    // exclusive prefix sum in place: four counters per lane and iteration, one warp scan of the lane totals
    uint32_t carry = 0;
    for (uint32_t c0 = 0; c0 < 32768u; c0 += 128u) {
        const uint32_t ci = c0 + 4u * (uint32_t)lane;
        uint32_t v[4], t = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) { v[j] = simt::ldg_cg_u32(g.end + ci + j); t += v[j]; }
        uint32_t xs = t;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = simt::shfl(HCW_FULL, xs, lane >= d ? lane - d : lane); if (lane >= d) xs += y; }
        uint32_t run = xs - t + carry;
#pragma unroll
        for (int j = 0; j < 4; j++) { simt::stg_u32(g.end + ci + j, run); run += v[j]; }
        carry += simt::shfl(HCW_FULL, xs, 31);
    }
    simt::syncwarp(HCW_FULL);
    // stable scatter, 32 consecutive positions per step: the lanes sharing a hash are found with MATCH.ANY, the lowest
    // adds the group's size, the others take their places behind it.  Afterwards end[h] = the end of bucket h.
    for (int base8 = lo; base8 < hi; base8 += 256) {
        uint32_t hh[8];
#pragma unroll
        for (int j = 0; j < 8; j++) { const int p = base8 + 32 * j + lane; hh[j] = p < hi ? simt::ldg_u16(g.rank + (p - B)) : 0xFFFFFFFFu; }
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int base = base8 + 32 * j;
            if (base >= hi) break;
            const int p = base + lane;
            const bool act = p < hi;
            const uint32_t h = hh[j];
            const uint32_t same = simt::match_any(HCW_FULL, h);
            const int leader = simt::ffs(same) - 1;
            uint32_t first = 0;
            if (act && lane == leader) first = simt::atomg_add(g.end + h, (uint32_t)simt::popc(same));
            first = simt::shfl(HCW_FULL, first, leader);
            const uint32_t idx = first + (uint32_t)simt::popc(same & ((1u << lane) - 1u));
            if (act) { simt::stg_u16(g.sorted + idx, (uint32_t)(p - B)); simt::stg_u16(g.rank + (p - B), idx); }
            simt::syncwarp(HCW_FULL);
        }
    }
    simt::syncwarp(HCW_FULL);
}

// ---- the segmented index: the members hcw_search, hcw_scan and hcw_parse use (see HcwIndex) ----------------------------
// q's place in the index: its rank in its segment (q >> 16), the entries of its bucket below it in that segment and the end
// of its bucket in the segment before
struct HcwwAt {
    int r, a, e1;
    SIMT_MEM HcwwAt shfl(int l) const
    {
        return HcwwAt{(int)simt::shfl(HCW_FULL, (uint32_t)r, l), (int)simt::shfl(HCW_FULL, (uint32_t)a, l),
                      (int)simt::shfl(HCW_FULL, (uint32_t)e1, l)};
    }
};

struct HcwwIndex {
    typedef HcwwAt At;
    HcwwSeg seg0, seg1;           // segment s lives in seg0 (s even) / seg1 (s odd)
    int held0, held1;             // the segment each slot holds (-1: none)
    // (selected, not indexed: an indexed array of them would live in local memory)
    SIMT_MEM HcwwSeg seg(int s) const { return (s & 1) ? seg1 : seg0; }
    SIMT_MEM int held(int s) const { return (s & 1) ? held1 : held0; }
    SIMT_MEM void hold(int s) { if (s & 1) held1 = s; else held0 = s; }

    SIMT_MEM At at(const HcwBlock<false>& w, int q) const
    {
        const uint32_t h = hcw_hash(w.rd32((uint32_t)q));
        At a;
        const int s = q >> 16;
        const HcwwSeg g = seg(s);
        a.r = (int)simt::ldg_u16(g.rank + (q & 0xFFFF));
        a.a = a.r - (h ? (int)simt::ldg_cg_u32(g.end + h - 1) : 0);
        a.e1 = s ? (int)simt::ldg_cg_u32(seg(s - 1).end + h) : 0;
        return a;
    }
    // candidate k of q (k < 257): a position, or -1 where the walk has left q's window.  Entries of the previous segment
    // below q's bucket come back as positions too: the caller's hash test ends the walk there.
    SIMT_MEM int cand(const At& a, int q, int k) const
    {
        const int s = q >> 16;
        if (k < a.a) return (s << 16) + (int)simt::ldg_u16(seg(s).sorted + (a.r - 1 - k));
        const int idx = a.e1 - 1 - (k - a.a);
        if (!s || idx < 0) return -1;
        const int p = ((s - 1) << 16) + (int)simt::ldg_u16(seg(s - 1).sorted + idx);
        return p >= q - 65535 ? p : -1;
    }
    SIMT_MEM bool ends_at_0(int q) const { return q < HCWW_SEG; }                // only a walk from segment 0 reaches it
    // segments s and s - 1 of q resident (warp-uniform q; searches never go down, so neither is built twice)
    SIMT_MEM void prepare(const HcwBlock<false>& w, int q)
    {
        const int s = q >> 16;
        if (s >= 1 && held(s - 1) != s - 1) { hcww_build(w, seg(s - 1), s - 1); hold(s - 1); }
        if (held(s) != s) { hcww_build(w, seg(s), s); hold(s); }
    }
    // a scan round stays in one segment
    SIMT_MEM int round_end(int ip, int mflimit) const
    {
        int end = ((ip >> 16) + 1) << 16;
        if (end > ip + 64) end = ip + 64;
        return end < mflimit ? end : mflimit;
    }
};

// One block of more than 64 KiB, all 32 lanes.  `index` = this warp's HCWW_INDEX_BYTES.  Returns what hcw_parse returns;
// HCW_FALLBACK also for a block of at most 64 KiB.
SIMT_DEV int hcww_encode_block(void* index, const uint8_t* src, int n, uint8_t* dst, int cap, int lane)
{
    if (n < 0 || cap < 0) return 0;
    if (n <= HCW_MAX_BLOCK) return HCW_FALLBACK;
    HcwBlock<false> w;
    w.src = src; w.n = n; w.lane = lane; w.in.init(src);
    w.mflimit = n - 12; w.matchlimit = n - 5;
    w.v0 = w.rd32(0);
    HcwwIndex x;
    uint8_t* ix = (uint8_t*)index;
    x.seg0.rank = (uint16_t*)ix;                    x.seg0.sorted = x.seg0.rank + 65536; x.seg0.end = (uint32_t*)(x.seg0.sorted + 65536);
    x.seg1.rank = (uint16_t*)(ix + HCWW_SEG_BYTES); x.seg1.sorted = x.seg1.rank + 65536; x.seg1.end = (uint32_t*)(x.seg1.sorted + 65536);
    x.held0 = x.held1 = -1;
    return hcw_parse(w, x, dst, cap);
}

}  // namespace lz4b200
