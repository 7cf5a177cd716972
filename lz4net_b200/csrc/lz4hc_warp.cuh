// lz4hc_warp.cuh -- byte-exact LZ4HC r93 encoder for blocks of at most 64 KiB, ONE WARP per block, no pointer chasing.
//
// Replaces LZ4_compressHC_limitedOutput (original/lz4hc.c:358-755; lz4net: src/LZ4ps/LZ4Codec.Safe64HC.Dirty.cs:71-522)
// for the block size BASELINE configs[2] names.  The thread-per-block kernel (lz4hc_encode.cuh) stays for larger blocks
// and for the rare blocks this one hands back (HCW_FALLBACK).
//
// The observation the design rests on: in a block of <= 64 KiB the reference's hash chains do not depend on the parse.
// LZ4HC_Insert (:358-373) inserts EVERY position below the searched one, in order, so chain[p] is the distance from p to
// the previous position with the same 15-bit hash (or to position 0, where the zero-filled heads point, :332), whatever
// was matched before.  A chain walk from position q (:423-433, :477-514) therefore visits
//     the positions < q of q's hash bucket in descending order, then position 0, then stops
// (chain[0] = 0xFFFF leads below ip - 65535; no delta is clamped and no slot aliases in 64 KiB).  So the warp
//   1. BUILDS the index once per block: a stable counting sort of the positions by hash (`sorted`, bucket by bucket in
//      ascending position) and each position's place in it (`rank`) -- histogram and stable scatter with atomics on
//      packed u16 counters (in shared memory, or in the warp's arena slot), 32 positions per step;
//   2. searches by GATHER: the candidates of q are sorted[rank[q]-1], sorted[rank[q]-2], ... -- consecutive entries, one
//      coalesced load for 32 of them, scored by the 32 lanes at once (common length / backward extension per lane, the
//      reference's "first candidate that beats everything before it" = first maximum, one REDUX);
//   3. scans literal stretches 64 positions per round, a lane per position (the index is static: no insert hazard).
// The 3-match look-ahead parse (:557-742) and LZ4_encodeSequence (:521-550) are control flow over those searches and are
// restated branch for branch, warp-uniformly.  The search, the scan and the parse are written against a small index
// interface (HcwIndex below); lz4hc_window.cuh runs the same three on its segmented index for blocks above 64 KiB.
//
// The two places where r93's state DOES depend on the parse are detected and the block is handed to the exact scalar
// kernel (HCW_FALLBACK; both are conservative, neither has been seen on the test corpora except when constructed):
//   * the repeat detector (:411-420, :437-455) rewrites chain[ip..end) to the period `delta` <= 4.  That equals the
//     static distance unless two of the period's `delta` strings share a hash (then a colliding position sits between p and
//     p - delta); the heads it skips are re-established by the run's last period.  delta >= 2 checks the <= 4 hashes.
//   * a search below a position that has already been inserted would see later positions in the real chain; the parse
//     never does that (every wider match covers its search position), the kernel checks it anyway.
#pragma once
#include "simt.cuh"
#include "lz4_copy.cuh"

namespace lz4b200 {

constexpr int    HCW_MAX_BLOCK   = 65536;
// per warp in flight: rank[65536] + sorted[65536] (u16) + the build's bucket counters (u16[32768]; only used by the
// variant that keeps nothing in shared memory)
constexpr size_t HCW_INDEX_BYTES = 2u * 65536u * sizeof(uint16_t) + 32768u * sizeof(uint16_t);
constexpr int    HCW_SMEM_BYTES  = 65536 + 16;                        // SMEM variant: bucket counters during the build, then the block's bytes
constexpr int    HCW_FALLBACK    = (int)0x80000000;                   // out_len marker: this block needs the scalar kernel
constexpr uint32_t HCW_FULL      = 0xFFFFFFFFu;

// Two placements of the block's bytes and of the build's counters, same code otherwise:
//   SMEM = true : both in 64 KiB of shared memory (counters first, then the staged block): candidate bytes at LDS latency,
//                 three warps (blocks) per SM;
//   SMEM = false: the block is read through the read-only path (L1 / L2), the counters live in the warp's arena slot
//                 (global atomics): no shared memory, as many warps per SM as the launch asks for.
// HcwBlock is the block as the search, the scan and the parse read it (lz4hc_window.cuh uses it with SMEM = false).
template <bool SMEM>
struct HcwBlock {
    simt::smem_ref sm;            // SMEM: HCW_SMEM_BYTES
    InWords in;                   // the input through aligned 32-bit words (the build; !SMEM: every read)
    const uint8_t* src; int n, lane, mflimit, matchlimit;
    uint32_t v0;                  // the four bytes at position 0 (the end of every walk that reaches it)

    // four bytes / one byte at position p of the block (p + 3 < n)
    SIMT_MEM uint32_t rd32(uint32_t p) const
    {
        if (SMEM) { const uint32_t q = p & ~3u; return simt::funnel_r(simt::lds_u32(sm, q), simt::lds_u32(sm, q + 4), (p & 3u) * 8u); }
        return in.at((int)p);
    }
    SIMT_MEM uint32_t rd8(uint32_t p) const { return SMEM ? simt::lds_u8(sm, p) : (uint32_t)simt::ldg_nc_u8(src + p); }
};

// The build's bucket counters: u16, two to a word, word w at byte 4w (SMEM: at the start of the shared memory; !SMEM: the
// 16384 words at `cnt`)
template <bool SMEM>
struct HcwCounters {
    simt::smem_ref sm;
    uint32_t* cnt;
    int lane;
    SIMT_MEM void cnt_zero() const
    {
        if (SMEM) for (uint32_t i = (uint32_t)lane * 16u; i < 65536u; i += 512u) simt::sts_v4(sm, i, uint4{0, 0, 0, 0});
        else      for (uint32_t i = (uint32_t)lane * 4u; i < 16384u; i += 128u) simt::stg_v4(cnt + i, uint4{0, 0, 0, 0});
    }
    SIMT_MEM uint32_t cnt_add(uint32_t h) const                      // bucket h's counter += 1, returns the old counter
    {
        const uint32_t inc = (h & 1u) ? 0x10000u : 1u;
        const uint32_t o = SMEM ? simt::atoms_add(sm, (h >> 1) * 4u, inc) : simt::atomg_add(cnt + (h >> 1), inc);
        return (o >> ((h & 1u) * 16u)) & 0xFFFFu;
    }
    SIMT_MEM uint32_t cnt_add_n(uint32_t h, uint32_t n) const          // += n (global counters), returns the old counter
    {
        const uint32_t o = simt::atomg_add(cnt + (h >> 1), (h & 1u) ? (n << 16) : n);
        return (o >> ((h & 1u) * 16u)) & 0xFFFFu;
    }
    SIMT_MEM uint32_t cnt_get(uint32_t h) const
    {
        if (SMEM) return simt::lds_u16(sm, h * 2u);
        return (simt::ldg_cg_u32(cnt + (h >> 1)) >> ((h & 1u) * 16u)) & 0xFFFFu;        // (L2: the word is modified by atomics)
    }
    SIMT_MEM uint32_t cnt_word(uint32_t wi) const { return SMEM ? simt::lds_u32(sm, wi * 4u) : simt::ldg_cg_u32(cnt + wi); }
    SIMT_MEM void cnt_word_set(uint32_t wi, uint32_t v) const { if (SMEM) simt::sts_u32(sm, wi * 4u, v); else simt::stg_u32(cnt + wi, v); }
};

SIMT_DEV uint32_t hcw_hash(uint32_t v) { return (v * 2654435761u) >> 17; }                   // :245-246 HASH_LOG 15

// The static index of a block of <= 64 KiB (built by hcw_build): candidate k of q is sorted[rank[q]-1-k] while that entry
// is in q's bucket, then position 0.  The search, the scan and the parse reach an index only through these members
// (lz4hc_window.cuh's HcwwIndex is the other implementation):
//   At                   q's place in the index, with shfl(l) = lane l's place
//   at(w, q)             q's place
//   cand(at, q, k)       candidate k of q: a position, or -1 for none
//   ends_at_0(q)         whether the walk from q ends at position 0 once its candidates run out
//   prepare(w, q)        before a scan round at q and before a wider search at q (warp-uniform q)
//   round_end(ip, mfl)   the end of the scan round that starts at ip
struct HcwAt {                    // q's place in the index: rank[q]
    int r;
    SIMT_MEM HcwAt shfl(int l) const { return HcwAt{(int)simt::shfl(HCW_FULL, (uint32_t)r, l)}; }
};

struct HcwIndex {
    typedef HcwAt At;
    uint16_t* rank;               // rank[p]: index of position p in `sorted` (positions 1 .. mflimit-1)
    uint16_t* sorted;             // positions ordered by (hash, position)

    template <bool SMEM>
    SIMT_MEM At at(const HcwBlock<SMEM>&, int q) const { return At{(int)simt::ldg_u16(rank + q)}; }
    // candidate k of q: a position, or -1 below the first entry.  An entry of another bucket comes back as a position:
    // the caller's hash test ends the walk there.
    SIMT_MEM int cand(const At& a, int, int k) const { const int idx = a.r - 1 - k; return idx >= 0 ? (int)simt::ldg_u16(sorted + idx) : -1; }
    SIMT_MEM bool ends_at_0(int) const { return true; }                             // every walk ends at position 0
    template <bool SMEM>
    SIMT_MEM void prepare(const HcwBlock<SMEM>&, int) {}                       // (the whole index is built up front)
    SIMT_MEM int round_end(int ip, int mflimit) const { return ip + 64 < mflimit ? ip + 64 : mflimit; }
};

// equal bytes of [a..) and [b..), a < limit  (== the 8/4/2/1 scheme of :376-391); one lane
template <bool SMEM>
SIMT_DEV int hcw_common(const HcwBlock<SMEM>& w, int a, int b, int limit)
{
    const int a0 = a;
    while (a + 4 <= limit) {
        const uint32_t x = w.rd32((uint32_t)a) ^ w.rd32((uint32_t)b);
        if (x) return a - a0 + ((simt::ffs(x) - 1) >> 3);
        a += 4; b += 4;
    }
    while (a < limit && w.rd8((uint32_t)a) == w.rd8((uint32_t)b)) { a++; b++; }
    return a - a0;
}

// the same count by the whole warp for ONE pair (a, b, limit identical in every lane): 128 bytes per step, the first
// differing word found with one vote.  Same value as hcw_common (the common prefix, capped at limit).
template <bool SMEM>
SIMT_DEV int hcw_common_warp(const HcwBlock<SMEM>& w, int a, int b, int limit)
{
    for (int done = 0; ; done += 128) {
        const int pa = a + done + 4 * w.lane;
        const bool in = pa + 4 <= limit;
        const uint32_t x = in ? (w.rd32((uint32_t)pa) ^ w.rd32((uint32_t)(b + done + 4 * w.lane))) : 0u;
        const uint32_t m = simt::ballot(HCW_FULL, !in || x != 0u);
        if (m) {
            const int f = simt::ffs(m) - 1;
            const uint32_t xf = simt::shfl(HCW_FULL, x, f);
            int t = a + done + 4 * f;                                  // (lane f's position)
            if (t + 4 <= limit) return t - a + ((simt::ffs(xf) - 1) >> 3);
            while (t < limit && w.rd8((uint32_t)t) == w.rd8((uint32_t)(b + t - a))) t++;     // fewer than four bytes left
            return t - a;
        }
    }
}

// literal source: the staged block (position 0 at shared offset 0, so alignment = position alignment)
struct HcwSmemSrc {
    static constexpr bool PIPELINED = false;
    simt::smem_ref sm; uint32_t at;
    SIMT_MEM uint8_t byte(uint32_t i) const { return (uint8_t)simt::lds_u8(sm, at + i); }
    SIMT_MEM uint32_t misalign(uint32_t i) const { return (at + i) & 15u; }
    SIMT_MEM uint4 word(uint32_t i, int k) const { return simt::lds_v4(sm, ((at + i) & ~15u) + 16u * (uint32_t)k); }
};

// the same through the read-only path (not pipelined: the warp's registers are worth more as resident warps here)
struct HcwInputSrc {
    static constexpr bool PIPELINED = false;
    const uint8_t* p;
    SIMT_MEM uint8_t byte(uint32_t i) const { return simt::ldg_nc_u8(p + i); }
    SIMT_MEM uint32_t misalign(uint32_t i) const { return (uint32_t)((uintptr_t)(p + i) & 15); }
    SIMT_MEM uint4 word(uint32_t i, int k) const { return simt::ldg_nc_v4((const uint8_t*)(((uintptr_t)(p + i)) & ~(uintptr_t)15) + 16 * k); }
};

// ---- 1. the index ---------------------------------------------------------------------------------------------------
template <bool SMEM>
SIMT_DEV void hcw_build(const HcwBlock<SMEM>& w, const HcwIndex& x, const HcwCounters<SMEM>& ct)
{
    const int lane = w.lane, P = w.mflimit;                               // positions 1 .. P-1 are ever searched or walked to
    const InWords& in = w.in;
    ct.cnt_zero();
    simt::syncwarp(HCW_FULL);
    // bucket sizes: u16 counters, two to a word, atomic adds on the word (a bucket never holds 65536 positions: no carry).
    // 128 positions per iteration, their input words requested together; the hashes are parked in rank[] for the scatter.
    for (int base = 1; base < P; base += 128) {
        InWords::Raw raw[4];
#pragma unroll
        for (int j = 0; j < 4; j++) { const int p = base + 32 * j + lane; if (p < P) raw[j] = in.raw<0>(p); }      // p <= n - 13: both words hold input bytes
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int p = base + 32 * j + lane;
            if (p < P) { const uint32_t h = hcw_hash(InWords::word(raw[j])); simt::stg_u16(x.rank + p, h); ct.cnt_add(h); }
        }
    }
    simt::syncwarp(HCW_FULL);
    // exclusive prefix sum in place: counter -> first index of the bucket.  Eight counters (four words) per lane and
    // iteration: lane-local prefix, one warp scan of the lane totals.
    uint32_t carry = 0;
    for (uint32_t w0 = 0; w0 < 16384u; w0 += 128u) {
        const uint32_t wi = w0 + 4u * (uint32_t)lane;
        uint32_t v[4], s = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) { v[j] = ct.cnt_word(wi + j); s += (v[j] & 0xFFFFu) + (v[j] >> 16); }
        uint32_t xs = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = simt::shfl(HCW_FULL, xs, lane >= d ? lane - d : lane); if (lane >= d) xs += y; }
        uint32_t run = xs - s + carry;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t lo = v[j] & 0xFFFFu, hi = v[j] >> 16;
            ct.cnt_word_set(wi + j, (run & 0xFFFFu) | ((run + lo) << 16));
            run += lo + hi;
        }
        carry += simt::shfl(HCW_FULL, xs, 31);
    }
    simt::syncwarp(HCW_FULL);
    // stable scatter, 32 consecutive positions per step (eight steps' hashes requested together)
    for (int base8 = 1; base8 < P; base8 += 256) {
        uint32_t hh[8];
#pragma unroll
        for (int j = 0; j < 8; j++) { const int p = base8 + 32 * j + lane; hh[j] = p < P ? simt::ldg_u16(x.rank + p) : 0xFFFFFFFFu; }
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int base = base8 + 32 * j;
            if (base >= P) break;
            const int p = base + lane;
            const bool act = p < P;
            const uint32_t h = hh[j];
            uint32_t idx;
            if (SMEM) {
                // counters at LDS / ATOMS latency: every lane adds for itself; lanes that share a hash inside the step get
                // their indices from the atomic in no particular order, so such a step (one lane sees a counter that is not
                // the value every lane read before) re-ranks the sharing lanes by position
                const uint32_t c0 = act ? ct.cnt_get(h) : 0u;
                simt::syncwarp(HCW_FULL);
                idx = c0;
                if (act) idx = ct.cnt_add(h);
                uint32_t pend = simt::ballot(HCW_FULL, act && idx != c0);
                while (pend) {
                    const uint32_t hl = simt::shfl(HCW_FULL, h, simt::ffs(pend) - 1);
                    const uint32_t same = simt::ballot(HCW_FULL, h == hl);
                    if (h == hl) idx = c0 + (uint32_t)simt::popc(same & ((1u << lane) - 1u));
                    pend &= ~same;
                }
            } else {
                // counters an L2 round trip away: the lanes that share a hash are found first (MATCH.ANY is cheaper than a
                // second round trip), the lowest of them adds the group's size, the others take their place behind it
                const uint32_t same = simt::match_any(HCW_FULL, h);
                const int leader = simt::ffs(same) - 1;
                uint32_t first = 0;
                if (act && lane == leader) first = ct.cnt_add_n(h, (uint32_t)simt::popc(same));
                first = simt::shfl(HCW_FULL, first, leader);
                idx = first + (uint32_t)simt::popc(same & ((1u << lane) - 1u));
            }
            if (act) { simt::stg_u16(x.sorted + idx, (uint32_t)p); simt::stg_u16(x.rank + p, idx); }
            simt::syncwarp(HCW_FULL);
        }
    }
}

// the block's bytes into shared memory (aligned 16-byte reads of words that hold at least one input byte)
SIMT_DEV void hcw_stage(const HcwBlock<true>& w)
{
    for (uint32_t i = (uint32_t)w.lane * 16u; i < (uint32_t)w.n; i += 512u) {
        const uintptr_t a = (uintptr_t)(w.src + i), al = a & ~(uintptr_t)15;
        const uint32_t r = (uint32_t)(a & 15);
        uint4 v = simt::ldg_nc_v4((const void*)al);
        if (r) {
            uint4 hi = uint4{0, 0, 0, 0};
            if (al + 16 < (uintptr_t)(w.src + w.n)) hi = simt::ldg_nc_v4((const void*)(al + 16));
            v = shift16(v, hi, r);
        }
        simt::sts_v4(w.sm, i, v);
    }
    simt::syncwarp(HCW_FULL);
}

// ---- 2. one search, the candidates scored 32 at a time ----------------------------------------------------------------
struct HcwHit { int len, ref, start, repl, delta; };

// WIDER = false: LZ4HC_InsertAndFindBestMatch (:394-459) at q (len 0 = no match).
// WIDER = true : LZ4HC_InsertAndGetWiderMatch (:462-518) at q with start_limit / longest; len <= longest = nothing better.
// `at` = x.at(w, q).  Candidate k is x.cand(at, q, k) while that position is in q's bucket, then position 0 where the
// index says the walk ends there, then nothing; at most 256 are examined (:403, :471), one more when the first one lies
// within 4 bytes (:411-420 consumes it without an attempt).  The reference's byte filters (:426, :480) only skip
// candidates that cannot win; the 4-byte test implies them.
template <bool WIDER, bool SMEM, class X>
SIMT_DEV HcwHit hcw_search(const HcwBlock<SMEM>& w, const X& x, int q, const typename X::At& at, int start_limit, int longest)
{
    const int lane = w.lane;
    const uint32_t vq = w.rd32((uint32_t)q), h = hcw_hash(vq);
    uint32_t best = 0, best_c = 0, best_back = 0;
    int K = 256;
    HcwHit out{0, 0, 0, 0, 0};
    for (int b0 = 0; ; b0 += 4) {
        int cc[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {                                     // four batches requested at once
            const int k = 32 * (b0 + j) + lane;
            cc[j] = k < 257 ? x.cand(at, q, k) : -1;
        }
        bool ended = false;
#pragma unroll 1
        for (int j = 0; j < 4 && !ended; j++) {                           // (one copy of the scoring code: the kernel is large enough)
            const int k = 32 * (b0 + j) + lane;
            int c = j == 0 ? cc[0] : (j == 1 ? cc[1] : (j == 2 ? cc[2] : cc[3]));
            uint32_t vc = 0;
            bool inb = false;
            if (c >= 0 && k < K) { vc = w.rd32((uint32_t)c); inb = hcw_hash(vc) == h; }
            const uint32_t outm = simt::ballot(HCW_FULL, !inb);
            const int first_out = outm ? simt::ffs(outm) - 1 : 32;
            bool valid = lane < first_out;
            if (lane == first_out && k < K && x.ends_at_0(q)) { valid = true; c = 0; vc = w.v0; }    // the walk ends at position 0
            if (!WIDER && b0 == 0 && j == 0) {
                // (lane 0 is valid unless the walk ends before its first candidate: then neither K nor the repeat
                // detector below is used)
                const int c_first = (int)simt::shfl(HCW_FULL, (uint32_t)c, 0);
                if (c_first >= q - 4) K = 257;
            }
            uint32_t key = 0, back = 0;
            const bool eq = valid && vc == vq;
            const uint32_t eqm = simt::ballot(HCW_FULL, eq);
            if (eqm && !(eqm & (eqm - 1u))) {
                // one matching candidate in the batch (sparse data): the whole warp counts its length, 128 bytes a step
                const int f = simt::ffs(eqm) - 1;
                const int cf = (int)simt::shfl(HCW_FULL, (uint32_t)c, f);
                uint32_t len = 4u + (uint32_t)hcw_common_warp(w, q + 4, cf + 4, w.matchlimit);
                if (WIDER) {                                              // :505 backwards, a lane per byte
                    int lim = q - start_limit; if (cf < lim) lim = cf;    // steps allowed: startt > startLimit, reft > base
                    uint32_t bk = 0;
                    for (int done = 0; done < lim; done += 32) {
                        const int i = done + w.lane;
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
                    int lim = q - start_limit; if (c < lim) lim = c;      // steps allowed: startt > startLimit, reft > base
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
            if (!WIDER && b0 == 0 && j == 0) {                            // :411-420 repeat detector: candidate 0, <= 4 back, matching
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

// ---- 3. literal scan: the first position in [ip, end) (end = x.round_end(ip, mflimit)) whose walk holds a match ---------
// Every lane walks for its own two positions (ip+lane, ip+32+lane), four candidates per memory round trip.  Returns the
// offset of the first position with a match (a position has one iff some examined candidate has its four bytes: every
// such candidate yields >= 4, :428-431) or -1, and that position's place in the index.
template <class At>
struct HcwScan { int off; At at; };

template <bool SMEM, class X>
SIMT_DEV HcwScan<typename X::At> hcw_scan(const HcwBlock<SMEM>& w, const X& x, int ip, int end)
{
    typedef typename X::At At;
    const int lane = w.lane;
    int q[2]; bool act[2]; At at[2];
    int cand[2][4];
#pragma unroll
    for (int s = 0; s < 2; s++) {
        q[s] = ip + 32 * s + lane; act[s] = q[s] < end;
        at[s] = act[s] ? x.at(w, q[s]) : At{};
    }
#pragma unroll
    for (int s = 0; s < 2; s++)
#pragma unroll
        for (int t = 0; t < 4; t++) cand[s][t] = act[s] ? x.cand(at[s], q[s], t) : -1;
    HcwScan<At> res{-1, At{}};
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const uint32_t vq = act[s] ? w.rd32((uint32_t)q[s]) : 0u, h = hcw_hash(vq);
        int k = 0, K = 256;
        bool done = !act[s], hit = false;
        for (;;) {
#pragma unroll
            for (int t = 0; t < 4; t++) {
                if (!done) {
                    int c = cand[s][t];
                    uint32_t vc = 0;
                    bool inb = false;
                    if (c >= 0) { vc = w.rd32((uint32_t)c); inb = hcw_hash(vc) == h; }
                    if (!inb) {
                        if (x.ends_at_0(q[s])) { c = 0; vc = w.v0; }
                        else done = true;                                 // the walk is over without a match
                    }
                    if (!done) {
                        if (k == 0 && c >= q[s] - 4) K = 257;
                        if (vc == vq) { hit = true; done = true; }
                        else if (!inb) done = true;
                        else if (++k >= K) done = true;
                    }
                }
            }
            const uint32_t hits = simt::ballot(HCW_FULL, hit), und = simt::ballot(HCW_FULL, !done);
            const uint32_t below = hits ? ((1u << (simt::ffs(hits) - 1)) - 1u) : HCW_FULL;
            if (!(und & below)) {
                if (hits) { const int l = simt::ffs(hits) - 1; res.off = 32 * s + l; res.at = at[s].shfl(l); }
                break;
            }
#pragma unroll
            for (int t = 0; t < 4; t++) cand[s][t] = !done ? x.cand(at[s], q[s], k + t) : -1;
        }
        if (res.off >= 0) break;
    }
    return res;
}

// ---- output ---------------------------------------------------------------------------------------------------------
struct HcwOut {
    uint8_t* dst; int cap, op, ip, anchor, lane;
    SIMT_MEM void put(int at, uint32_t v) const { if (lane == 0 && at < cap) simt::stg_u8(dst + at, (uint8_t)v); }   // never outside [dst, dst+cap)
};

SIMT_DEV int hcw_put_len(const HcwOut& o, int at, int v)               // 255, 255, ..., v % 255
{
    const int n255 = v / 255;
    for (int i = o.lane; i < n255; i += 32) if (at + i < o.cap) simt::stg_u8(o.dst + at + i, 255);
    o.put(at + n255, (uint32_t)(v - 255 * n255));
    return at + n255 + 1;
}

// the literals [at, at+n) of the block -> dst (the caller has checked that they fit).  Runs of HC sequences are short:
// byte steps inline; the 128-bit mover (incompressible stretches, the last literals) is ONE out-of-line copy of its code.
SIMT_NOINLINE void hcw_copy_long_smem(uint8_t* dst, simt::smem_ref sm, uint32_t at, uint32_t n, int lane)
{
    group_copy<32, false>(dst, HcwSmemSrc{sm, at}, n, lane, HCW_FULL);
}
SIMT_NOINLINE void hcw_copy_long_input(uint8_t* dst, const uint8_t* src, uint32_t n, int lane)
{
    group_copy<32, false>(dst, HcwInputSrc{src}, n, lane, HCW_FULL);
}
template <bool SMEM>
SIMT_DEV void hcw_literals(const HcwBlock<SMEM>& w, uint8_t* dst, int at, int n)
{
    if (n < 64) {
        for (int i = w.lane; i < n; i += 32) simt::stg_u8(dst + i, (uint8_t)w.rd8((uint32_t)(at + i)));
        return;
    }
    if (SMEM) hcw_copy_long_smem(dst, w.sm, (uint32_t)at, (uint32_t)n, w.lane);
    else      hcw_copy_long_input(dst, w.src + at, (uint32_t)n, w.lane);
}

template <bool SMEM>
SIMT_DEV bool hcw_emit(const HcwBlock<SMEM>& w, HcwOut& o, int ml, int ref)       // :521-550 LZ4_encodeSequence; true = output full
{
    const int L = o.ip - o.anchor, tok = o.op++;
    uint32_t tv;
    if (o.op + L + 8 + (L >> 8) > o.cap) return true;                  // :529 (token, length bytes, literals and offset fit from here on)
    if (L >= 15) { tv = 0xF0; o.op = hcw_put_len(o, o.op, L - 15); } else tv = (uint32_t)L << 4;
    hcw_literals(w, o.dst + o.op, o.anchor, L);
    o.op += L;
    o.put(o.op, (uint32_t)(o.ip - ref) & 255); o.put(o.op + 1, ((uint32_t)(o.ip - ref) >> 8) & 255); o.op += 2;
    const int len = ml - 4;
    if (o.op + 6 + (L >> 8) > o.cap) return true;                      // :541 -- the LITERAL length, as the reference does
    if (len >= 15) { tv |= 15; o.op = hcw_put_len(o, o.op, len - 15); } else tv |= (uint32_t)len;
    o.put(tok, tv);
    o.ip += ml; o.anchor = o.ip;
    return false;
}

// ---- 4. the parse (:581-739) over either index, all 32 lanes ----------------------------------------------------------
// Returns the bytes written, 0 = did not fit, HCW_FALLBACK = a state the index does not describe (the same value in every
// lane).  x.prepare(w, q) runs before every scan round at q and every wider search at q.
template <bool SMEM, class X>
SIMT_DEV int hcw_parse(const HcwBlock<SMEM>& w, X& x, uint8_t* dst, int cap)
{
    const int lane = w.lane, n = w.n, mflimit = w.mflimit;
    HcwOut o{dst, cap, 0, 1, 0, lane};                                 // :581 ip = 1
    int next = 1;                                                      // nextToUpdate (:334)
    int ml, ml2, ml3, ml0, ref = 0, ref2 = 0, ref3 = 0, ref0, start2 = 0, start3 = 0, start0;
    bool odd = false;                                                  // a state the index does not describe

    while (o.ip < mflimit) {                                           // :584
        if (o.ip < next) return HCW_FALLBACK;
        x.prepare(w, o.ip);
        const int end = x.round_end(o.ip, mflimit);
        const HcwScan<typename X::At> sc = hcw_scan(w, x, o.ip, end);
        if (sc.off < 0) { next = end - 1; o.ip = end; continue; }     // (end - ip) x "if (!ml) { ip++; continue; }"
        o.ip += sc.off;
        next = o.ip;
        {
            const HcwHit b = hcw_search<false>(w, x, o.ip, sc.at, 0, 0);
            ml = b.len; ref = b.ref;
            if (b.repl) {                                              // :437-455: chain[ip..end) := delta, nextToUpdate = end
                if (b.delta >= 2) {                                    // equal to the static chain unless two of the period's strings share a hash
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
        // The look-ahead (:594-726) as a loop with ONE wider search per turn (one copy of the search code): a turn is
        // either _Search2 or _Search3; _Search2 falling through into _Search3 is "next turn, _Search3".
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
                x.prepare(w, wq);
                const HcwHit h = hcw_search<true>(w, x, wq, x.at(w, wq), wlim, wlong);
                wml = h.len; wref = h.ref; wstart = h.start;
            }
            if (to_search2) {                                          // _Search2  :594-622
                ml2 = wml; if (wml > wlong) { ref2 = wref; start2 = wstart; }
                if (ml2 == ml) { if (hcw_emit(w, o, ml, ref)) return 0; break; }
                if (start0 < o.ip && start2 < o.ip + ml0) { o.ip = start0; ref = ref0; ml = ml0; }
                if (start2 - o.ip < 3) { ml = ml2; o.ip = start2; ref = ref2; continue; }
                to_search2 = false; continue;                          // on to _Search3
            }
            // _Search3  :648-726
            ml3 = wml; if (wml > wlong) { ref3 = wref; start3 = wstart; }
            if (ml3 == ml2) {                                          // :648-657 two sequences
                if (start2 < o.ip + ml) ml = start2 - o.ip;
                if (hcw_emit(w, o, ml, ref)) return 0;
                o.ip = start2;
                if (hcw_emit(w, o, ml2, ref2)) return 0;
                break;
            }
            if (start3 < o.ip + ml + 3) {                              // :659-691
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
                continue;                                              // _Search3 again
            }
            if (start2 < o.ip + ml) {                                  // :695-714
                if (start2 - o.ip < 15) {
                    if (ml > 18) ml = 18;
                    if (o.ip + ml > start2 + ml2 - 4) ml = (start2 - o.ip) + ml2 - 4;
                    const int corr = ml - (start2 - o.ip);
                    if (corr > 0) { start2 += corr; ref2 += corr; ml2 -= corr; }
                } else ml = start2 - o.ip;
            }
            if (hcw_emit(w, o, ml, ref)) return 0;                     // :715
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

// One block of at most 64 KiB, all 32 lanes.  `sm` = HCW_SMEM_BYTES of shared memory (SMEM variant), `index` = this warp's
// HCW_INDEX_BYTES.  Returns what hcw_parse returns; HCW_FALLBACK also for a block above 64 KiB.
template <bool SMEM>
SIMT_DEV int hcw_encode_block(simt::smem_ref sm, void* index, const uint8_t* src, int n, uint8_t* dst, int cap, int lane)
{
    if (n < 0 || cap < 0) return 0;
    if (n > HCW_MAX_BLOCK) return HCW_FALLBACK;
    HcwBlock<SMEM> w; w.sm = sm;
    w.src = src; w.n = n; w.lane = lane; w.in.init(src);
    w.mflimit = n - 12; w.matchlimit = n - 5;
    HcwIndex x; x.rank = (uint16_t*)index; x.sorted = x.rank + 65536;
    if (w.mflimit > 1) hcw_build(w, x, HcwCounters<SMEM>{sm, (uint32_t*)(x.sorted + 65536), lane});
    if constexpr (SMEM) hcw_stage(w);
    w.v0 = n >= 4 ? w.rd32(0) : 0u;
    return hcw_parse(w, x, dst, cap);
}

}  // namespace lz4b200
