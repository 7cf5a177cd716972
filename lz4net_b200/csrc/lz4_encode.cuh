// lz4_encode.cuh -- byte-exact LZ4 r93 fast encoder, one warp per block.
//
// Replaces LZ4_compress64kCtx (original/lz4.c:573-771; lz4net: LZ4_compress64kCtx_safe64,
// src/LZ4ps/LZ4Codec.Safe64.Dirty.cs:306-527) for inputs < 65547 bytes and LZ4_compressCtx (original/lz4.c:345-562;
// Safe64.Dirty.cs:77-300) above that, behind the LZ4_compress_limitedOutput dispatch (original/lz4.c:774-792).
// The emitted bytes must equal lz4net's LZ4Codec.Encode, so the greedy parse is reproduced exactly -- but as a
// warp-wide formulation of the serial state machine (SURVEY.md Appendix A), split in two phases:
//
// PARSE (the serial dependency chain, kept as short as it can be):
//   * one "round" evaluates 32 consecutive iterations of the reference's find-match loop at once: the probe
//     positions follow from the attempt counter alone (step = attempts >> 6, :636/:644), their hashes only depend on
//     the input, and the table state each serial iteration would have seen is reconstructed inside the round with
//     MATCH.ANY (a lower lane with the same hash supplies the candidate instead of the table);
//   * VOTE + FFS picks the first lane that either hits or runs past mflimit (:648); only lanes up to it commit their
//     table update, highest lane per bucket winning -- exactly the serial write order;
//   * the two table operations that follow every match (insert ip-2, probe+insert ip, :739-751) are not a separate
//     step: they ride in lanes 0 and 1 of the next round ("fused round"), whose remaining 30 lanes are the first 30
//     iterations of the find-match loop that starts at ip+1.  A hit in lane 1 is the reference's zero-literal
//     `goto _next_match`;
//   * the forward match-length count (:701-716) starts at ip + 4 as the round found it.  The backward catch-up (:657)
//     is not on this chain: it moves ip and ref back together over matching bytes, so the match end mp, the offset and
//     everything the next round needs (org = mp - 2, anchor = mp, the mflimit test) are the same without it;
//   * nothing is written during the parse: each found sequence is one record (anchor, literal length up to the ip the
//     round found, offset, match length from there) parked in the registers of one lane.
// EMIT (every 32 sequences, fully lane-parallel):
//   * catch-up: lane k moves sequence k's split point back, 4 bytes per word compare; the rare catch-ups longer than a
//     few words finish with the whole warp on one sequence, 32 bytes per step;
//   * sizes -> warp prefix sum -> every sequence's output position; the reference's output-limit checks (:663, :728,
//     :762) are evaluated for all 32 sequences at once from those positions;
//   * lane k writes token, length bytes and offset of sequence k; literal runs are copied by the whole warp, four
//     short runs per step.
//
// The 16 KiB position table (u16[8192] for the 64 K variant, u32[4096] for the general one -- the same footprint)
// lives in shared memory, zero-filled per block (zero == "candidate at position 0", :583/:651).  The input is read
// through the read-only path; the lines ahead of the cursor are software-prefetched (the parse is a latency chain:
// a cold miss on the forward stream would stall it for a full DRAM round trip per 128 bytes).
#pragma once
#include "simt.cuh"
#include "lz4_copy.cuh"
#include "enc_prof.cuh"

namespace lz4b200 {

struct alignas(16) EncShared { uint32_t table[4096]; };

constexpr int LZ4_64KLIMIT = 65547;                                // original/lz4.c:565

// Heuristics that only steer which (equivalent) code path runs -- never the emitted bytes.
struct EncTune {
    int pf_dist = 0;          // > 0: L1 prefetch that many bytes ahead; < 0: L2; 0: off
    int lane_copy_max = 12;   // emission: every lane copies its own literal run when all 32 runs are at most this long
    int probe_max = 8;        // after a literal run shorter than this, the post-match probe is tried alone before a round
    int wide_min = 24;        // after a literal run at least this long, the fused round is 64 iterations wide
};

// flags kept above the 16-bit offset of a parked sequence
constexpr uint32_t SEQ_NOCHK = 0x10000u;                           // zero-literal `goto _next_match` sequence: no :663 check
constexpr uint32_t SEQ_LAST  = 0x20000u;                           // the last literal run (no match part)

// A long literal run (> 32 bytes), copied by the whole warp with pipelined 128-bit moves.  Kept out of line: it is the
// rare path of the emission, and inlined its eight vector registers pairs would spill the parse loop.
SIMT_NOINLINE void copy_long_literals(uint8_t* dst, const uint8_t* src, uint32_t n, int lane)
{
    InputSrc sp{src};
    group_copy<32, false>(dst, sp, n, lane, 0xFFFFFFFFu);
}

// The position table behind a 32-bit shared-window address.
template <bool GENERAL>
struct EncTable {
    simt::smem_ref r;
    SIMT_MEM void bind(void* table) { r = simt::smem_ref_of(table); }
    SIMT_MEM int  get(uint32_t h) const { return GENERAL ? (int)simt::lds_u32(r, h * 4u) : (int)simt::lds_u16(r, h * 2u); }
    SIMT_MEM void put(uint32_t h, int pos) const { if (GENERAL) simt::sts_u32(r, h * 4u, (uint32_t)pos); else simt::sts_u16(r, h * 2u, (uint32_t)pos); }
};

// One round = W*32 consecutive serial iterations of the find-match loop; lane l evaluates iterations l and (W == 2) 32+l.
// Positions are a pure function of the attempt number a (>= 65): step(a) = a >> 6 (:636/:644), so the position of
// attempt a is org + S(a) with S(a) = sum_{j<a} (j >> 6) = q * (32*(q-1) + (a & 63)), q = a >> 6 -- `org` stays the
// same from round to round until the next match.
//
// The candidate of a serial iteration is the table entry -- unless an earlier iteration of this same round has the same
// hash, in which case it is that iteration's position.  Sharing is found through the table itself while the candidate
// words (fetched for the table entries at once) are in flight: every iteration writes its index into its bucket and
// reads it back; one that does not find its own index ("lost") shares the bucket with the winner.  The losers write
// once more: now the winner learns about a loser, and a loser that loses again knows the bucket has three or more
// sharers.  Two sharers (by far the common case: a match whose source lies inside the round) are resolved exactly from
// that -- the later iteration's candidate is the earlier one's position and its candidate word is the earlier one's
// input word, moved by SHFL, no load; three or more take the exact path (one vote per hash bit and half) over all the
// iterations of the round, so its result is final as well.  At the end every bucket gets its final value: the position
// of the last sharer whose iteration really ran (index <= f), or its old entry if none did.
// f: the first iteration that hits or runs past mflimit; 32*W when none does.
struct RoundOut { int f; bool finished; int ip, ref; };

// SIMPLE: every attempt of the round still has step 1 and lies inside the block (known from two warp-uniform tests):
// positions are consecutive and every iteration is valid.
template <bool GENERAL, int W, int DUP, int LDP, bool SIMPLE>
SIMT_DEV RoundOut find_round(const EncTable<GENERAL>& T, const InWords& in, int org, uint32_t A0, bool fused,
                             int mflimit, int lane, uint32_t lt_mask)
{
    constexpr uint32_t FULL = 0xFFFFFFFFu;
    constexpr int HSHIFT = GENERAL ? 20 : 19;                      // :185-187 / :566-569
    ENC_PROF_T0(tp);
    ENC_PROF_EVENT(EP_ROUND);
    ENC_PROF_EVENT_IF(EP_ROUND_WIDE, W == 2);
    int pos[W]; bool valid[W]; uint32_t v[W], h[W]; int t[W]; uint32_t vmask[W];
    InWords::Raw rp[W], rc[W];
    const int p0 = org + (int)A0 - 64;                             // SIMPLE: attempt A0 + i sits at p0 + i (S(a) = a - 64 up to a = 128)
#pragma unroll
    for (int s = 0; s < W; s++) {
        const bool special = fused && s == 0 && lane < 2;          // fused round: lane 0 = insert ip-2, lane 1 = probe+insert ip
        if (SIMPLE) { pos[s] = p0 + 32 * s + lane; valid[s] = true; }
        else {
            const uint32_t a = A0 + 32u * s + (uint32_t)lane, q = a >> 6;
            pos[s] = org + (int)(q * (((q - 1u) << 5) + (a & 63u)));
            valid[s] = special || pos[s] + (int)q <= mflimit;      // the bounds test precedes the probe (:420 / :648)
        }
        if (special && lane == 0) pos[s] -= 1;                     // (the formula gives ip-1 and ip for attempts 65 and 66)
    }
#pragma unroll
    for (int s = 0; s < W; s++) rp[s] = in.raw<LDP>(valid[s] ? pos[s] : 0);
#pragma unroll
    for (int s = 0; s < W; s++) vmask[s] = SIMPLE ? FULL : simt::ballot(FULL, valid[s]);
#pragma unroll
    for (int s = 0; s < W; s++) { v[s] = InWords::word(rp[s]); h[s] = (v[s] * 2654435761u) >> HSHIFT; }
#pragma unroll
    for (int s = 0; s < W; s++) t[s] = T.get(h[s]);
#pragma unroll
    for (int s = 0; s < W; s++) rc[s] = in.raw<LDP>(t[s]);          // candidate words for the table entries: in flight from here
    ENC_PROF_LAP(EP_C_LOADHASH, tp);

    RoundOut o; o.finished = false; o.ip = o.ref = 0;
    int partner[W];
    uint32_t anylost = 0u, multi = 0u;
#pragma unroll
    for (int s = 0; s < W; s++) partner[s] = -1;
    if (DUP == 2) {
        simt::syncwarp(FULL);                                      // every lane has read its buckets
#pragma unroll
        for (int s = 0; s < W; s++) if (valid[s]) T.put(h[s], 32 * s + lane);
        simt::syncwarp(FULL);
        int r1[W]; bool lost[W]; bool anyl = false;
#pragma unroll
        for (int s = 0; s < W; s++) { r1[s] = valid[s] ? T.get(h[s]) : 32 * s + lane; lost[s] = r1[s] != 32 * s + lane; anyl = anyl || lost[s]; }
        anylost = simt::ballot(FULL, anyl);
        if (anylost) {
            simt::syncwarp(FULL);
#pragma unroll
            for (int s = 0; s < W; s++) if (lost[s]) T.put(h[s], 32 * s + lane);
            simt::syncwarp(FULL);
            bool m = false;
#pragma unroll
            for (int s = 0; s < W; s++) {
                const int r2 = valid[s] ? T.get(h[s]) : 32 * s + lane;
                if (lost[s]) { partner[s] = r1[s]; m = m || r2 != 32 * s + lane; }
                else if (r2 != 32 * s + lane) partner[s] = r2;
            }
            multi = simt::ballot(FULL, m);
        }
    }
    ENC_PROF_LAP(EP_C_SAMEHASH, tp);
    if (DUP == 2 && multi == 0u) {
        ENC_PROF_EVENT_IF(EP_PAIR, anylost != 0u);
        uint32_t hitm[W]; int cand[W];
#pragma unroll
        for (int s = 0; s < W; s++) {
            cand[s] = t[s];
            uint32_t pv = 0; bool lowerp = false;
            if (anylost) {                                          // the earlier sharer's position and input word
                const int pl = partner[s] >= 0 ? (partner[s] & 31) : lane;
                int pp; pv = simt::shfl(FULL, v[0], pl);
                if (SIMPLE) pp = p0 + partner[s] - ((fused && partner[s] == 0) ? 1 : 0);     // a position follows from its index
                else pp = (int)simt::shfl(FULL, (uint32_t)pos[0], pl);
                if (W == 2) {
                    const uint32_t pv1 = simt::shfl(FULL, v[W - 1], pl);
                    if (!SIMPLE) { const int pp1 = (int)simt::shfl(FULL, (uint32_t)pos[W - 1], pl); if (partner[s] >= 32) pp = pp1; }
                    if (partner[s] >= 32) pv = pv1;
                }
                lowerp = partner[s] >= 0 && partner[s] < 32 * s + lane;
                if (lowerp) cand[s] = pp;
            }
            simt::tie(rc[s].lo, anylost | multi);                   // wait for the candidate words only after the votes above
            const uint32_t w = lowerp ? pv : InWords::word(rc[s]);
            const bool hit = valid[s] && !(fused && s == 0 && lane == 0) &&           // (lane 0 of a fused round only inserts)
                             (!GENERAL || cand[s] >= pos[s] - 65535) && w == v[s];    // :429 / :654, :531 / :751
            hitm[s] = simt::ballot(FULL, hit);
        }
        // valid iterations are a prefix of the round (positions grow); the first event is a hit or the first invalid one
        int nv = simt::popc(vmask[0]), fh = hitm[0] ? simt::ffs(hitm[0]) - 1 : 64;
        if (W == 2) { nv += simt::popc(vmask[W - 1]); if (!hitm[0] && hitm[W - 1]) fh = 32 + simt::ffs(hitm[W - 1]) - 1; }
        const int f = fh < nv ? fh : nv;                            // == 32*W: nothing happened in this round
        simt::syncwarp(FULL);                                      // every lane's read-backs are done before any bucket is rewritten
        // final bucket values: the last sharer whose iteration ran (index <= f) leaves its position, else the old entry.
        // Without a partner I write either way; of two sharers the later one writes if it ran, the earlier one if the
        // later one did not (its own position if it ran itself, else the old entry).
#pragma unroll
        for (int s = 0; s < W; s++) {
            const int me = 32 * s + lane; const bool ran = me <= f;
            const bool wr = valid[s] && (partner[s] < 0 || (partner[s] > me ? (!ran || partner[s] > f) : ran));
            if (wr) T.put(h[s], ran ? pos[s] : t[s]);
        }
        simt::syncwarp(FULL);
        o.f = f;
        if (f < 32 * W) {
            if (fh >= nv) o.finished = true;                        // ran past mflimit -> last literals (:420 / :648)
            else {
                const bool hi = W == 2 && f >= 32;
                o.ip = SIMPLE ? p0 + f : (int)simt::shfl(FULL, (uint32_t)(hi ? pos[W - 1] : pos[0]), f & 31);   // (f == 0 never hits in a fused round)
                o.ref = (int)simt::shfl(FULL, (uint32_t)(hi ? cand[W - 1] : cand[0]), f & 31);
            }
        }
        ENC_PROF_LAP(EP_C_VOTE, tp);
        return o;
    }
    // ---- exact path over the whole round (three or more iterations share a bucket, or DUP == 1) ----
    if (DUP == 2) {
        simt::syncwarp(FULL);
#pragma unroll
        for (int s = 0; s < W; s++) if (valid[s]) T.put(h[s], t[s]);    // (all sharers read the same old entry)
        simt::syncwarp(FULL);
    }
    {
        // same[s][u]: the lanes whose iteration in half u has the hash of my iteration in half s (invalid ones: nobody)
        uint32_t same[W][W];
#pragma unroll
        for (int s = 0; s < W; s++)
#pragma unroll
            for (int u = 0; u < W; u++) same[s][u] = vmask[u];
#pragma unroll
        for (int b = 0; b < (GENERAL ? 12 : 13); b++) {
            uint32_t vb[W];
#pragma unroll
            for (int u = 0; u < W; u++) vb[u] = simt::ballot(FULL, (h[u] >> b) & 1u);
#pragma unroll
            for (int s = 0; s < W; s++)
#pragma unroll
                for (int u = 0; u < W; u++) same[s][u] &= ((h[s] >> b) & 1u) ? vb[u] : ~vb[u];
        }
        // the candidate: the position of the latest earlier sharer (in my half, else in the first), else the table entry
        int cand[W]; uint32_t stop[W];
#pragma unroll
        for (int s = 0; s < W; s++) {
            const uint32_t own = valid[s] ? same[s][s] & lt_mask : 0u;
            const uint32_t lower = own ? own : (s == 1 && valid[s] ? same[W - 1][0] : 0u);
            const int from = lower ? 31 - simt::clz(lower) : lane;
            int fwd = (int)simt::shfl(FULL, (uint32_t)pos[0], from);
            uint32_t fv = simt::shfl(FULL, v[0], from);
            if (s == 1) {
                const int fwd1 = (int)simt::shfl(FULL, (uint32_t)pos[W - 1], from);
                const uint32_t fv1 = simt::shfl(FULL, v[W - 1], from);
                if (own) { fwd = fwd1; fv = fv1; }
            }
            cand[s] = lower ? fwd : t[s];
            const uint32_t w = lower ? fv : InWords::word(rc[s]);
            const bool hit = valid[s] && !(fused && s == 0 && lane == 0) && (!GENERAL || cand[s] >= pos[s] - 65535) && w == v[s];
            stop[s] = simt::ballot(FULL, !valid[s] || hit);
        }
        int f = stop[0] ? simt::ffs(stop[0]) - 1 : 32;
        if (W == 2 && !stop[0]) f = stop[W - 1] ? 32 + simt::ffs(stop[W - 1]) - 1 : 64;
        // commit the table writes of the serial iterations that really happened (index <= f), last writer per bucket
        uint32_t cmask[W];
#pragma unroll
        for (int u = 0; u < W; u++) {
            const int fu = f - 32 * u;
            cmask[u] = fu < 0 ? 0u : (fu >= 31 ? vmask[u] : (vmask[u] & ((2u << fu) - 1u)));
        }
#pragma unroll
        for (int s = 0; s < W; s++) {
            uint32_t later = same[s][s] & cmask[s] & ~((2u << lane) - 1u);
            if (s == 0 && W == 2) later |= same[0][W - 1] & cmask[W - 1];
            if (valid[s] && ((cmask[s] >> lane) & 1u) && !later) T.put(h[s], pos[s]);
        }
        simt::syncwarp(FULL);
        o.f = f;
        if (f < 32 * W) {
            const bool hi = W == 2 && f >= 32;
            if (!((cmask[hi ? W - 1 : 0] >> (f & 31)) & 1u)) o.finished = true;
            else {
                o.ip = (int)simt::shfl(FULL, (uint32_t)(hi ? pos[W - 1] : pos[0]), f & 31);
                o.ref = (int)simt::shfl(FULL, (uint32_t)(hi ? cand[W - 1] : cand[0]), f & 31);
            }
        }
        ENC_PROF_EVENT(EP_EXACT);
        ENC_PROF_LAP(EP_C_EXACT, tp);
        return o;
    }
}

template <bool GENERAL, int DUP, int LDP>
SIMT_DEV int encode_block_t(void* table, const uint8_t* src, int n, uint8_t* dst, int cap, int lane, EncTune tune)
{
    constexpr uint32_t FULL = 0xFFFFFFFFu;
    const int mflimit = n - 12, matchlimit = n - 5;                // :361,:366 / :590,:596
    const uint32_t lt_mask = (1u << lane) - 1u;
    ENC_PROF_T0(tb);
    ENC_PROF_T0(tp);
    ENC_PROF_EVENT(EP_BLOCK);
    InWords in; in.init(src);
    EncTable<GENERAL> T; T.bind(table);

    // sequence queue: lane k holds record k
    int q = 0, op = 0;
    int sq_anchor = 0, sq_L = 0, sq_M = 0; uint32_t sq_off = 0;

    // ---- EMIT: write out the q queued sequences; false = the output does not fit (the reference returns 0) ----------
    const uint64_t spol = LDP == 1 ? simt::l2_policy_stream() : 0;
    auto st8 = [&](uint8_t* p, uint32_t v) { if (LDP == 1) simt::stg_hint_u8(p, v, spol); else simt::stg_u8(p, (uint8_t)v); };
    auto flush = [&]() -> bool {
        ENC_PROF_EVENT(EP_FLUSH);
        const bool act = lane < q;
        int L = sq_L, M = sq_M;
        const bool last = (sq_off & SEQ_LAST) != 0, nochk = (sq_off & SEQ_NOCHK) != 0;
        // ---- catch up (:432 / :657), lane k for sequence k.  Parked as found: ip = anchor + L, ref = ip - offset.  Word
        // compares backwards, 4 bytes per step and lane; the few catch-ups longer than CU_LANE_STEPS words finish with
        // the whole warp on one sequence at a time, 32 bytes per step.  ip - c >= anchor and ref - c >= 0 bound c.
        {
            constexpr int CU_LANE_STEPS = 4;
            const int ip = sq_anchor + L, ref = ip - (int)(sq_off & 0xFFFFu);
            const int lim = L < ref ? L : ref;
            int c = 0;
            bool go = act && !last && lim > 0;
#pragma unroll 1
            for (int s = 0; s < CU_LANE_STEPS && simt::ballot(FULL, go); s++) {
                if (go) {
                    const uint32_t x = in.back(ip - c) ^ in.back(ref - c);
                    const int e = x ? simt::clz(x) >> 3 : 4;
                    c += e;
                    go = e == 4 && c < lim;
                }
            }
            for (uint32_t lg = simt::ballot(FULL, go); lg; lg &= lg - 1u) {
                const int k = simt::ffs(lg) - 1;
                const int ipk = (int)simt::shfl(FULL, (uint32_t)ip, k), refk = (int)simt::shfl(FULL, (uint32_t)ref, k);
                const int limk = (int)simt::shfl(FULL, (uint32_t)lim, k);
                int ck = (int)simt::shfl(FULL, (uint32_t)c, k);
                ENC_PROF_EVENT(EP_CATCHUP_LONG);
                for (;;) {
                    const int j = ck + lane + 1;
                    const bool eq = j <= limk && simt::ldg_nc_u8(src + (ipk - j)) == simt::ldg_nc_u8(src + (refk - j));
                    const uint32_t ne = ~simt::ballot(FULL, eq);
                    const int e = ne ? simt::ffs(ne) - 1 : 32;
                    ck += e;
                    if (e < 32) break;
                }
                if (lane == k) c = ck;
            }
            if (c > lim) c = lim;
            L -= c; M += c;
        }
        ENC_PROF_LAP(EP_C_CATCHUP, tp);
        const int extL = L >= 15 ? 1 + (L - 15) / 255 : 0;
        const int extM = (!last && M >= 15) ? 1 + (M - 15) / 255 : 0;
        const int size = act ? 1 + extL + L + (last ? 0 : 2 + extM) : 0;
        int incl = size;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int t = (int)simt::shfl(FULL, (uint32_t)incl, lane >= d ? lane - d : lane);
            if (lane >= d) incl += t;
        }
        const int start = op + incl - size;
        bool bad = false;
        if (act) {
            if (last) bad = start + L + 1 + (L - 15 + 255) / 255 > cap;                       // :540 / :762
            else {
                if (!nochk) bad = start + 1 + L + (L >> 8) > cap - 8;                         // :438 / :663
                bad = bad || start + 1 + extL + L + 2 + (M >> 8) > cap - 6                    // :501 / :728
                          || start + size > cap;                   // (only reachable with run lengths beyond any 64 KiB block)
            }
        }
        if (simt::ballot(FULL, bad)) return false;
        int litpos = 0;
        if (act) {
            const int lt = L < 15 ? L : 15, mt = last ? 0 : (M < 15 ? M : 15);
            st8(dst + start, (uint32_t)((lt << 4) | mt));
            int o = start + 1;
            if (L >= 15) { int v = L - 15; for (; v >= 255; v -= 255) st8(dst + o++, 255u); st8(dst + o++, (uint32_t)v); }
            litpos = o; o += L;
            if (!last) {
                st8(dst + o, sq_off & 0xFFu); st8(dst + o + 1, (sq_off >> 8) & 0xFFu);       // :470 / :695
                o += 2;
                if (M >= 15) { int v = M - 15; for (; v >= 255; v -= 255) st8(dst + o++, 255u); st8(dst + o++, (uint32_t)v); }
            }
        }
        // literal runs.  All short (token-dense data): every lane copies its own run, byte by byte -- a handful of
        // iterations for 32 sequences.  Otherwise the whole warp copies run after run, four short runs per step.
        const int Lq = act ? L : 0;
        const int Lmax = (int)simt::reduce_max(FULL, (uint32_t)Lq);
        if (Lmax <= tune.lane_copy_max) {
            const uint8_t* sp = src + sq_anchor; uint8_t* dp = dst + litpos;
            for (int i = 0; i < Lq; i++) st8(dp + i, simt::ldg_nc_u8(sp + i));
        } else
        for (int s = 0; s < q; s += 4) {
            int a[4], d[4], l[4];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                a[i] = (int)simt::shfl(FULL, (uint32_t)sq_anchor, (s + i) & 31);
                d[i] = (int)simt::shfl(FULL, (uint32_t)litpos, (s + i) & 31);
                l[i] = (s + i) < q ? (int)simt::shfl(FULL, (uint32_t)Lq, (s + i) & 31) : 0;
            }
            const int l01 = l[0] > l[1] ? l[0] : l[1], l23 = l[2] > l[3] ? l[2] : l[3];
            if ((l01 > l23 ? l01 : l23) <= 32) {
                uint8_t b[4];
#pragma unroll
                for (int i = 0; i < 4; i++) b[i] = lane < l[i] ? simt::ldg_nc_u8(src + a[i] + lane) : (uint8_t)0;
#pragma unroll
                for (int i = 0; i < 4; i++) if (lane < l[i]) st8(dst + d[i] + lane, b[i]);
            } else {
#pragma unroll 1
                for (int i = s; i < s + 4 && i < q; i++) {
                    const uint8_t* const sp = src + (int)simt::shfl(FULL, (uint32_t)sq_anchor, i);
                    uint8_t* const dp = dst + (int)simt::shfl(FULL, (uint32_t)litpos, i);
                    ENC_PROF_EVENT(EP_LONG_LIT);
                    copy_long_literals(dp, sp, simt::shfl(FULL, (uint32_t)Lq, i), lane);
                }
            }
        }
        op += (int)simt::shfl(FULL, (uint32_t)incl, 31);
        q = 0;
        ENC_PROF_LAP(EP_C_EMIT, tp);
        return true;
    };

    for (int i = lane; i < 1024; i += 32) ((uint4*)table)[i] = uint4{0, 0, 0, 0};
    simt::syncwarp(FULL);
    ENC_PROF_RESTART(tp);

    int anchor = 0;
    if (n >= 13) {                                                 // :387 / :615 (MINLENGTH)
        // Round state: attempt a sits at position org + S(a).  The find-match loop starts with attempt 67
        // (findMatchAttempts = (1 << 6) + 3, :409 / :636) at position `first`: org = first - S(67) = first - 3.
        // A fused round starts two attempts earlier: 65 and 66 are the post-match table operations on ip-2 and ip.
        int org = 1 - 3;                                           // :404 / :631: the first probe is at position 1
        uint32_t A0 = 67; bool fused = false, wide = false;
        bool probe_first = false;                                  // dense matches: try the post-match probe alone first
        int pfpos = 0;
        for (;;) {
            int ip = 0, ref = 0; bool again = false, have = false, finished = false;
            InWords::Raw pre_ra{0, 0, 0}, pre_rr{0, 0, 0}; bool pre = false;   // the first count words of a probe hit, already in flight
            if (probe_first) {
                // The post-match table operations (:519-531 / :739-751) on their own, warp-uniform: in token-dense data
                // the probe at ip usually hits (a zero-literal sequence) and a whole round would be wasted work.
                const int mp = anchor, p2 = mp - 2;
                const uint32_t v2 = in.at(p2), vi = in.at(mp);
                constexpr int HSHIFT = GENERAL ? 20 : 19;
                const uint32_t h2 = (v2 * 2654435761u) >> HSHIFT, h = (vi * 2654435761u) >> HSHIFT;
                const int t = (h == h2) ? p2 : T.get(h);
                const uint32_t w = in.at(t);
                // the words the match count will compare if the probe hits (it usually does here): requested together with the
                // candidate word, so the count does not start another memory round trip after the verdict
                {
                    const int a = mp + 4 + 4 * lane;
                    int room = matchlimit - a; room = room < 0 ? 0 : (room > 4 ? 4 : room);
                    pre_ra = in.raw<LDP>(room > 0 ? a : 0); pre_rr = in.raw<LDP>(room > 0 ? t + 4 + 4 * lane : 0);
                    pre = true;
                }
                simt::syncwarp(FULL);                              // every lane has read the bucket
                if (lane == 0) { T.put(h2, p2); T.put(h, mp); }
                simt::syncwarp(FULL);
                if ((!GENERAL || t > mp - 65536) && w == vi) { ip = mp; ref = t; again = true; have = true; }
                else { org = mp + 1 - 3; A0 = 67; fused = false; wide = false; pre = false; }
                ENC_PROF_EVENT(EP_PROBE);
                ENC_PROF_EVENT_IF(EP_PROBE_HIT, have);
                ENC_PROF_LAP(EP_C_PROBE, tp);
            }
            while (!have) {
                RoundOut r;
                const bool w2 = wide && DUP == 2;
                const int consumed = w2 ? 64 : 32;
                // step 1 up to attempt 128 (and 2 for attempt 128 itself), everything inside the block?
                const bool simple = A0 + (uint32_t)consumed - 1u <= 128u && org + (int)A0 - 64 + consumed + 1 <= mflimit;
                if (w2) r = simple ? find_round<GENERAL, 2, DUP, LDP, true>(T, in, org, A0, fused, mflimit, lane, lt_mask)
                                   : find_round<GENERAL, 2, DUP, LDP, false>(T, in, org, A0, fused, mflimit, lane, lt_mask);
                else    r = simple ? find_round<GENERAL, 1, DUP, LDP, true>(T, in, org, A0, fused, mflimit, lane, lt_mask)
                                   : find_round<GENERAL, 1, DUP, LDP, false>(T, in, org, A0, fused, mflimit, lane, lt_mask);
                if (r.f >= consumed) {                              // no hit: the find-match loop goes on
                    A0 += (uint32_t)consumed; fused = false; wide = true;
                    if (tune.pf_dist != 0) {                        // incompressible stretch: fetch what the round after next will read
                        const uint32_t qa = A0 >> 6;
                        const int p = org + (int)(qa * (((qa - 1u) << 5) + (A0 & 63u))) + 64 * (int)qa + 128 * lane;
                        if (lane < 8 && p < n) { if (tune.pf_dist > 0) simt::prefetch_l1(src + p); else simt::prefetch_l2(src + p); }
                    }
                    continue;
                }
                if (r.finished) { finished = true; break; }
                ip = r.ip; ref = r.ref; have = true;
                again = fused && r.f == 1;                          // zero-literal sequence (:531 / :751)
            }
            ENC_PROF_RESTART(tp);                                   // (the rounds count their own cycles)
            if (finished) break;

            // ---------------- count the match (:475-494 / :701-716) -------------------------------------------------
            // The backward catch-up (:657) is left to EMIT: it moves ip and ref back together over bytes that match, so
            // the match end mp, the offset and everything the next round needs are the same without it.
            int mp = ip + 4, mr = ref + 4;                          // forward cursors
            int cnt;
            {
                const int a = mp + 4 * lane;
                int room = matchlimit - a; room = room < 0 ? 0 : (room > 4 ? 4 : room);
                const InWords::Raw ra = pre ? pre_ra : in.raw<LDP>(room > 0 ? a : 0), rr = pre ? pre_rr : in.raw<LDP>(room > 0 ? mr + 4 * lane : 0);
                const uint32_t x = InWords::word(ra) ^ InWords::word(rr);
                cnt = x ? (simt::ffs(x) - 1) >> 3 : 4;
                if (cnt > room) cnt = room;
            }
            {
                uint32_t part = simt::ballot(FULL, cnt != 4);
                while (!part) {
                    // the first 128 bytes all matched: a long match.  Count 512 bytes per step, every load before the
                    // first vote (one memory round trip per 512 bytes)
                    mp += 128; mr += 128;
                    if (tune.pf_dist != 0 && lane < 4 && mp + 1024 + 128 * lane < n) simt::prefetch_l1(src + mp + 1024 + 128 * lane);
                    constexpr int NC = 4;
                    int c4[NC];
#pragma unroll
                    for (int k = 0; k < NC; k++) {
                        const int a = mp + 128 * k + 4 * lane;
                        int room = matchlimit - a; room = room < 0 ? 0 : (room > 4 ? 4 : room);
                        const uint32_t x = InWords::word(in.raw<LDP>(room > 0 ? a : 0)) ^ InWords::word(in.raw<LDP>(room > 0 ? mr + 128 * k + 4 * lane : 0));
                        c4[k] = x ? (simt::ffs(x) - 1) >> 3 : 4;
                        if (c4[k] > room) c4[k] = room;
                    }
#pragma unroll
                    for (int k = 0; k < NC; k++) {
                        if (part) break;
                        part = simt::ballot(FULL, c4[k] != 4);
                        if (part) cnt = c4[k]; else if (k < NC - 1) { mp += 128; mr += 128; }
                    }
                }
                const int pl = simt::ffs(part) - 1;
                mp += 4 * pl + (int)simt::shfl(FULL, (uint32_t)cnt, pl);
            }
            ENC_PROF_LAP(EP_C_COUNT, tp);
            // ---------------- park the sequence, not caught up (EMIT catches it up) ----------------
            const int L = ip - anchor;
            if (lane == q) {
                sq_anchor = anchor; sq_L = L; sq_M = mp - (ip + 4);
                sq_off = (uint32_t)(ip - ref) | (again ? SEQ_NOCHK : 0u);
            }
            ENC_PROF_EVENT(EP_SEQ);
            ENC_PROF_LAP(EP_C_PARK, tp);
            if (++q == 32 && !flush()) return 0;
            anchor = mp;
            if (mp > mflimit) break;                                // :516 / :736
            if (tune.pf_dist != 0 && mp + (tune.pf_dist > 0 ? tune.pf_dist : -tune.pf_dist) > pfpos && pfpos < n) {
                const int p = pfpos + 128 * lane;                   // keep the forward stream ahead of the cursor in cache
                if (lane < 4 && p < n) { if (tune.pf_dist > 0) simt::prefetch_l1(src + p); else simt::prefetch_l2(src + p); }
                pfpos += 512;
            }
            // What follows a match (:519-534 / :739-755): insert ip-2, probe + insert ip, then the find-match loop from
            // ip+1.  Short literal runs predict another immediate hit: do the probe alone first.  Otherwise all of it
            // is one fused round: attempts 65, 66 = ip-2, ip; 67.. = the loop.  S(66) = 2, so org = mp - 2.
            probe_first = L < tune.probe_max;                      // (L before the catch-up: at least the emitted one)
            org = mp - 2; A0 = 65; fused = true;
            wide = L >= tune.wide_min;                                      // long literal runs: the next match is probably > 30 bytes away
            ENC_PROF_LAP(EP_C_PARK, tp);
        }
    }

    // ---------------- last literals (:540-551 / :760-767) ----------------
    if (lane == q) { sq_anchor = anchor; sq_L = n - anchor; sq_off = SEQ_LAST; sq_M = 0; }
    ++q;
    ENC_PROF_EVENT(EP_SEQ);
    ENC_PROF_RESTART(tp);
    if (!flush()) return 0;
    ENC_PROF_LAP(EP_C_BLOCK, tb);
    return op;
}

// LZ4_compress_limitedOutput dispatch (original/lz4.c:774-792)
// `table`: 16 KiB of shared memory, 16-byte aligned, owned by this warp.
template <int DUP = 2, int LDP = 0>
SIMT_DEV int encode_block(void* table, const uint8_t* src, int n, uint8_t* dst, int cap, int lane, EncTune tune = EncTune{})
{
    if (n < 0 || cap < 0) return 0;
    simt::syncwarp(0xFFFFFFFFu);                                   // previous block's table users are done
    return n < LZ4_64KLIMIT ? encode_block_t<false, DUP, LDP>(table, src, n, dst, cap, lane, tune)
                            : encode_block_t<true, DUP, LDP>(table, src, n, dst, cap, lane, tune);
}

}  // namespace lz4b200
