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
// Search, scan and parse restate lz4hc_warp.cuh's for the segmented index; that header's kernels are left as they are
// (same instructions), its helpers (common length, output, sequence encoder) are used through a Hcw<false>.
#pragma once
#include "lz4hc_warp.cuh"

namespace lz4b200 {

constexpr int    HCWW_SEG         = 65536;
// per segment: rank u16[65536] + sorted u16[65536] + end u32[32768]; two segments per warp in flight
constexpr size_t HCWW_SEG_BYTES   = 2u * 65536u * sizeof(uint16_t) + 32768u * sizeof(uint32_t);
constexpr size_t HCWW_INDEX_BYTES = 2u * HCWW_SEG_BYTES;

struct HcwwSeg { uint16_t* rank; uint16_t* sorted; uint32_t* end; };

struct Hcww {
    Hcw<false> w;                 // the input, the lane, the limits (lz4hc_warp.cuh's helpers take it)
    HcwwSeg seg0, seg1;           // segment s lives in seg0 (s even) / seg1 (s odd)
    int held0, held1;             // the segment each slot holds (-1: none)
    // (selected, not indexed: an indexed array of them would live in local memory)
    SIMT_MEM HcwwSeg seg(int s) const { return (s & 1) ? seg1 : seg0; }
    SIMT_MEM int held(int s) const { return (s & 1) ? held1 : held0; }
    SIMT_MEM void hold(int s) { if (s & 1) held1 = s; else held0 = s; }
};

// ---- 1. the index, one segment -----------------------------------------------------------------------------------------
SIMT_DEV void hcww_build(const Hcww& x, int s)
{
    const HcwwSeg g = x.seg(s);
    const int lane = x.w.lane, B = s * HCWW_SEG;
    const int lo = B > 1 ? B : 1, hi = B + HCWW_SEG < x.w.mflimit ? B + HCWW_SEG : x.w.mflimit;   // positions 1 .. mflimit-1
    const InWords& in = x.w.in;
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

// segments s and s - 1 resident (warp-uniform s; searches never go down, so neither is built twice)
SIMT_DEV void hcww_need(Hcww& x, int s)
{
    if (s >= 1 && x.held(s - 1) != s - 1) { hcww_build(x, s - 1); x.hold(s - 1); }
    if (x.held(s) != s) { hcww_build(x, s); x.hold(s); }
}

// q's place in the index: its segment, rank there, the entries of its bucket below it in that segment and the end of its
// bucket in the segment before
struct HcwwAt { int s, r, a; int e1; };

SIMT_DEV HcwwAt hcww_at(const Hcww& x, int q, uint32_t h)
{
    HcwwAt at;
    at.s = q >> 16;
    const HcwwSeg g = x.seg(at.s);
    at.r = (int)simt::ldg_u16(g.rank + (q & 0xFFFF));
    at.a = at.r - (h ? (int)simt::ldg_cg_u32(g.end + h - 1) : 0);
    at.e1 = at.s ? (int)simt::ldg_cg_u32(x.seg(at.s - 1).end + h) : 0;
    return at;
}

// candidate k of q (k < 257): a position, or -1 where the walk has left q's window.  Entries of the previous segment below
// q's bucket come back as positions too: the caller's hash test ends the walk there, as it does in lz4hc_warp.cuh.
SIMT_DEV int hcww_cand(const Hcww& x, const HcwwAt& at, int q, int k)
{
    if (k < at.a) return (at.s << 16) + (int)simt::ldg_u16(x.seg(at.s).sorted + (at.r - 1 - k));
    const int idx = at.e1 - 1 - (k - at.a);
    if (!at.s || idx < 0) return -1;
    const int p = ((at.s - 1) << 16) + (int)simt::ldg_u16(x.seg(at.s - 1).sorted + idx);
    return p >= q - 65535 ? p : -1;
}

// ---- 2. one search (hcw_search on the segmented index) -------------------------------------------------------------------
template <bool WIDER>
SIMT_DEV HcwHit hcww_search(const Hcww& x, int q, int start_limit, int longest)
{
    const Hcw<false>& w = x.w;
    const int lane = w.lane;
    const uint32_t vq = w.rd32((uint32_t)q), h = hcw_hash(vq);
    const HcwwAt at = hcww_at(x, q, h);
    uint32_t best = 0, best_c = 0, best_back = 0;
    int K = 256;
    HcwHit out{0, 0, 0, 0, 0};
    for (int b0 = 0; ; b0 += 4) {
        int cc[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {                                     // four batches requested at once
            const int k = 32 * (b0 + j) + lane;
            cc[j] = k < 257 ? hcww_cand(x, at, q, k) : -1;
        }
        bool ended = false;
#pragma unroll 1
        for (int j = 0; j < 4 && !ended; j++) {
            const int k = 32 * (b0 + j) + lane;
            int c = j == 0 ? cc[0] : (j == 1 ? cc[1] : (j == 2 ? cc[2] : cc[3]));
            uint32_t vc = 0;
            bool inb = false;
            if (c >= 0 && k < K) { vc = w.rd32((uint32_t)c); inb = hcw_hash(vc) == h; }
            const uint32_t outm = simt::ballot(HCW_FULL, !inb);
            const int first_out = outm ? simt::ffs(outm) - 1 : 32;
            bool valid = lane < first_out;
            if (!valid) c = 0;
            if (lane == first_out && k < K && at.s == 0) { valid = true; vc = w.v0; }      // the walk ends at position 0 (q <= 65535)
            if (!WIDER && b0 == 0 && j == 0) {
                const int c_first = (int)simt::shfl(HCW_FULL, (uint32_t)c, 0);             // (an empty window: 0 < q - 4)
                if (c_first >= q - 4) K = 257;
            }
            uint32_t key = 0, back = 0;
            const bool eq = valid && vc == vq;
            const uint32_t eqm = simt::ballot(HCW_FULL, eq);
            if (eqm && !(eqm & (eqm - 1u))) {
                // one matching candidate in the batch: the whole warp counts its length, 128 bytes a step
                const int f = simt::ffs(eqm) - 1;
                const int cf = (int)simt::shfl(HCW_FULL, (uint32_t)c, f);
                uint32_t len = 4u + (uint32_t)hcw_common_warp(w, q + 4, cf + 4, w.matchlimit);
                if (WIDER) {                                              // :505 backwards, a lane per byte
                    int lim = q - start_limit; if (cf < lim) lim = cf;
                    uint32_t bk = 0;
                    for (int done = 0; done < lim; done += 32) {
                        const int i = done + lane;
                        const bool ok = i < lim && w.rd8((uint32_t)(q - 1 - i)) == w.rd8((uint32_t)(cf - 1 - i));
                        const uint32_t bad = simt::ballot(HCW_FULL, !ok);
                        if (bad) { bk = (uint32_t)(done + simt::ffs(bad) - 1); break; }
                        bk = (uint32_t)(done + 32);
                    }
                    back = bk; len += bk;
                }
                if (eq) key = len * 512u + (511u - (uint32_t)k);
            } else if (eq) {
                uint32_t len = 4u + (uint32_t)hcw_common(w, q + 4, c + 4, w.matchlimit);
                if (WIDER) {                                              // :505 backwards, four bytes at a time
                    int lim = q - start_limit; if (c < lim) lim = c;
                    bool open = true;
                    while (open && (int)back + 4 <= lim) {
                        const uint32_t d = w.rd32((uint32_t)q - back - 4u) ^ w.rd32((uint32_t)c - back - 4u);
                        if (d) { back += (uint32_t)simt::clz(d) >> 3; open = false; } else back += 4u;
                    }
                    while (open && (int)back < lim && w.rd8((uint32_t)q - back - 1u) == w.rd8((uint32_t)c - back - 1u)) back++;
                    len += back;
                }
                key = len * 512u + (511u - (uint32_t)k);                  // longest first, then earliest in the walk
            }
            const uint32_t bm = simt::reduce_max(HCW_FULL, key);
            if (bm > best) {
                const int holder = (int)((511u - (bm & 511u)) & 31u);
                best = bm;
                best_c = simt::shfl(HCW_FULL, (uint32_t)c, holder);
                if (WIDER) best_back = simt::shfl(HCW_FULL, back, holder);
            }
            if (!WIDER && b0 == 0 && j == 0) {                            // :411-420 repeat detector
                const uint32_t key0 = simt::shfl(HCW_FULL, key, 0);
                const int c_first = (int)simt::shfl(HCW_FULL, (uint32_t)c, 0);
                if (key0 && c_first >= q - 4) { out.repl = (int)(key0 >> 9); out.delta = q - c_first; }
            }
            if (first_out < 32) ended = true;
        }
        if (ended) break;
    }
    if (best) {
        const int len = (int)(best >> 9);
        if (!WIDER) { out.len = len; out.ref = (int)best_c; }
        else if (len > longest) { out.len = len; out.ref = (int)best_c - (int)best_back; out.start = q - (int)best_back; }
    }
    if (WIDER && out.len <= longest) out.len = longest;
    return out;
}

// ---- 3. literal scan: the first position in [ip, end) (end - ip <= 64, one segment) whose walk holds a match, or -1 ----
SIMT_DEV int hcww_scan(const Hcww& x, int ip, int end)
{
    const Hcw<false>& w = x.w;
    const int lane = w.lane;
    int q[2]; bool act[2]; uint32_t vq[2], h[2]; HcwwAt at[2];
    int cand[2][4];
#pragma unroll
    for (int s = 0; s < 2; s++) {
        q[s] = ip + 32 * s + lane; act[s] = q[s] < end;
        vq[s] = act[s] ? w.rd32((uint32_t)q[s]) : 0u; h[s] = hcw_hash(vq[s]);
    }
#pragma unroll
    for (int s = 0; s < 2; s++) at[s] = act[s] ? hcww_at(x, q[s], h[s]) : HcwwAt{0, 0, 0, 0};
#pragma unroll
    for (int s = 0; s < 2; s++)
#pragma unroll
        for (int t = 0; t < 4; t++) cand[s][t] = act[s] ? hcww_cand(x, at[s], q[s], t) : -1;
    int res = -1;
#pragma unroll
    for (int s = 0; s < 2; s++) {
        int k = 0, K = 256;
        bool done = !act[s], hit = false;
        for (;;) {
#pragma unroll
            for (int t = 0; t < 4; t++) {
                if (!done) {
                    int c = cand[s][t];
                    uint32_t vc = 0;
                    bool inb = false;
                    if (c >= 0) { vc = w.rd32((uint32_t)c); inb = hcw_hash(vc) == h[s]; }
                    if (!inb) {
                        if (at[s].s) done = true;                         // window exhausted (q > 65535: no position 0)
                        else { c = 0; vc = w.v0; }
                    }
                    if (!done) {
                        if (k == 0 && c >= q[s] - 4) K = 257;
                        if (vc == vq[s]) { hit = true; done = true; }
                        else if (!inb) done = true;
                        else if (++k >= K) done = true;
                    }
                }
            }
            const uint32_t hits = simt::ballot(HCW_FULL, hit), und = simt::ballot(HCW_FULL, !done);
            const uint32_t below = hits ? ((1u << (simt::ffs(hits) - 1)) - 1u) : HCW_FULL;
            if (!(und & below)) {
                if (hits) res = 32 * s + simt::ffs(hits) - 1;
                break;
            }
#pragma unroll
            for (int t = 0; t < 4; t++) cand[s][t] = !done ? hcww_cand(x, at[s], q[s], k + t) : -1;
        }
        if (res >= 0) break;
    }
    return res;
}

// One block of more than 64 KiB, all 32 lanes.  `index` = this warp's HCWW_INDEX_BYTES.  Returns the bytes written,
// 0 = did not fit, HCW_FALLBACK = not for this kernel (the same value in every lane).  The parse is hcw_encode_block's.
SIMT_DEV int hcww_encode_block(void* index, const uint8_t* src, int n, uint8_t* dst, int cap, int lane)
{
    if (n < 0 || cap < 0) return 0;
    if (n <= HCW_MAX_BLOCK) return HCW_FALLBACK;
    Hcww x;
    uint8_t* ix = (uint8_t*)index;
    x.seg0.rank = (uint16_t*)ix;                    x.seg0.sorted = x.seg0.rank + 65536; x.seg0.end = (uint32_t*)(x.seg0.sorted + 65536);
    x.seg1.rank = (uint16_t*)(ix + HCWW_SEG_BYTES); x.seg1.sorted = x.seg1.rank + 65536; x.seg1.end = (uint32_t*)(x.seg1.sorted + 65536);
    x.held0 = x.held1 = -1;
    Hcw<false>& w = x.w;
    w.rank = w.sorted = nullptr; w.cnt = nullptr;
    w.src = src; w.n = n; w.lane = lane; w.in.init(src);
    w.mflimit = n - 12; w.matchlimit = n - 5;
    w.v0 = w.rd32(0);
    HcwOut o{dst, cap, 0, 1, 0, lane};                                 // :581 ip = 1
    const int mflimit = w.mflimit;
    int next = 1;                                                      // nextToUpdate (:334)
    int ml, ml2, ml3, ml0, ref = 0, ref2 = 0, ref3 = 0, ref0, start2 = 0, start3 = 0, start0;
    bool odd = false;

    while (o.ip < mflimit) {                                           // :584
        if (o.ip < next) return HCW_FALLBACK;
        const int s = o.ip >> 16;
        hcww_need(x, s);
        int end = (s + 1) << 16;                                       // a scan round stays in one segment
        if (end > o.ip + 64) end = o.ip + 64;
        if (end > mflimit) end = mflimit;
        const int off = hcww_scan(x, o.ip, end);
        if (off < 0) { next = end - 1; o.ip = end; continue; }         // (end - ip) x "if (!ml) { ip++; continue; }"
        o.ip += off;
        next = o.ip;
        {
            const HcwHit b = hcww_search<false>(x, o.ip, 0, 0);
            ml = b.len; ref = b.ref;
            if (b.repl) {                                              // :437-455: chain[ip..end) := delta, nextToUpdate = end
                if (b.delta >= 2) {
                    const uint32_t hj = lane < b.delta ? hcw_hash(w.rd32((uint32_t)(o.ip - b.delta + lane))) : 0x10000u + (uint32_t)lane;
                    const uint32_t h0 = simt::shfl(HCW_FULL, hj, 0), h1 = simt::shfl(HCW_FULL, hj, 1), h2 = simt::shfl(HCW_FULL, hj, 2), h3 = simt::shfl(HCW_FULL, hj, 3);
                    if (h0 == h1 || h0 == h2 || h0 == h3 || h1 == h2 || h1 == h3 || h2 == h3) odd = true;
                }
                const int e = o.ip + b.repl - 3;
                if (e > next) next = e;
            }
        }
        if (odd || !ml) return HCW_FALLBACK;
        start0 = o.ip; ref0 = ref; ml0 = ml;                           // :589-592
        bool to_search2 = true;
        for (;;) {
            int wq, wlim, wlong;
            if (to_search2) { wq = o.ip + ml - 2; wlim = o.ip + 1; wlong = ml; }      // :595-597
            else {                                                     // :628-646
                if (start2 - o.ip < 18) {
                    int new_ml = ml > 18 ? 18 : ml;
                    if (o.ip + new_ml > start2 + ml2 - 4) new_ml = (start2 - o.ip) + ml2 - 4;
                    const int corr = new_ml - (start2 - o.ip);
                    if (corr > 0) { start2 += corr; ref2 += corr; ml2 -= corr; }
                }
                wq = start2 + ml2 - 3; wlim = start2; wlong = ml2;
            }
            int wml = wlong, wref = 0, wstart = 0;
            if (wq + (to_search2 ? 2 : 3) < mflimit) {                 // "ip + ml < mflimit" / "start2 + ml2 < mflimit"
                if (wq < next) return HCW_FALLBACK;
                next = wq;
                hcww_need(x, wq >> 16);
                const HcwHit hh = hcww_search<true>(x, wq, wlim, wlong);
                wml = hh.len; wref = hh.ref; wstart = hh.start;
            }
            if (to_search2) {                                          // _Search2  :594-622
                ml2 = wml; if (wml > wlong) { ref2 = wref; start2 = wstart; }
                if (ml2 == ml) { if (hcw_emit(w, o, ml, ref)) return 0; break; }
                if (start0 < o.ip && start2 < o.ip + ml0) { o.ip = start0; ref = ref0; ml = ml0; }
                if (start2 - o.ip < 3) { ml = ml2; o.ip = start2; ref = ref2; continue; }
                to_search2 = false; continue;
            }
            ml3 = wml; if (wml > wlong) { ref3 = wref; start3 = wstart; }             // _Search3  :648-726
            if (ml3 == ml2) {
                if (start2 < o.ip + ml) ml = start2 - o.ip;
                if (hcw_emit(w, o, ml, ref)) return 0;
                o.ip = start2;
                if (hcw_emit(w, o, ml2, ref2)) return 0;
                break;
            }
            if (start3 < o.ip + ml + 3) {
                if (start3 >= o.ip + ml) {
                    if (start2 < o.ip + ml) {
                        const int corr = o.ip + ml - start2;
                        start2 += corr; ref2 += corr; ml2 -= corr;
                        if (ml2 < 4) { start2 = start3; ref2 = ref3; ml2 = ml3; }
                    }
                    if (hcw_emit(w, o, ml, ref)) return 0;
                    o.ip = start3; ref = ref3; ml = ml3;
                    start0 = start2; ref0 = ref2; ml0 = ml2;
                    to_search2 = true; continue;
                }
                start2 = start3; ref2 = ref3; ml2 = ml3;
                continue;
            }
            if (start2 < o.ip + ml) {
                if (start2 - o.ip < 15) {
                    if (ml > 18) ml = 18;
                    if (o.ip + ml > start2 + ml2 - 4) ml = (start2 - o.ip) + ml2 - 4;
                    const int corr = ml - (start2 - o.ip);
                    if (corr > 0) { start2 += corr; ref2 += corr; ml2 -= corr; }
                } else ml = start2 - o.ip;
            }
            if (hcw_emit(w, o, ml, ref)) return 0;
            o.ip = start2; ref = ref2; ml = ml2;
            start2 = start3; ref2 = ref3; ml2 = ml3;
        }
    }
    {                                                                  // :729-739 last literals
        const int R = n - o.anchor;
        if ((uint32_t)(o.op + R + 1 + (R + 255 - 15) / 255) > (uint32_t)cap) return 0;
        if (R >= 15) { o.put(o.op++, 0xF0); o.op = hcw_put_len(o, o.op, R - 15); } else o.put(o.op++, (uint32_t)R << 4);
        hcw_literals(w, dst + o.op, o.anchor, R);
        o.op += R;
    }
    return o.op;
}

}  // namespace lz4b200
