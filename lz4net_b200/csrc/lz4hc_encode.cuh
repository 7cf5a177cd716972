// lz4hc_encode.cuh -- byte-exact LZ4HC r93 encoder, ONE THREAD per block.
//
// Replaces LZ4_compressHC_limitedOutput and its helpers (original/lz4hc.c:358-755; lz4net:
// src/LZ4ps/LZ4Codec.Safe64HC.Dirty.cs:71-522 behind Encode64HC, src/LZ4ps/LZ4Codec.Safe.cs:707-724).
//
// Why a thread and not a warp: the cost of HC is the hash-chain walk (<= 256 dependent hops per searched position,
// :423-433) -- pointer chasing whose next address is only known when the previous hop returns.  A warp cannot make
// one chain go faster; what a GPU can do is keep tens of thousands of independent chains in flight so that HBM/L2
// latency is hidden by thread-level parallelism.  Each thread therefore owns one block and a private
// 256 KiB state (heads u32[32768] + chain u16[65536], :231-237) in global memory, handed out from a scratch arena.
// The parse (3-match look-ahead state machine, :557-742) is control flow only and is restated branch for branch.
//
// Only chain[0] and the heads need initialising: every chain slot that a walk can reach was written by the insert
// of the position it describes (positions 1..next-1 are inserted contiguously, :358-373); slot 0 (position 0 is
// never inserted, :334) must read 0xFFFF so that walks reaching position 0 terminate.
#pragma once
#include "simt.cuh"
#include "lz4_copy.cuh"

namespace lz4b200 {

constexpr size_t HC_STATE_BYTES = 32768 * 4 + 65536 * 2;          // per block in flight

struct HcState {
    const uint8_t* src;
    uint32_t* heads;       // [32768] positions
    uint16_t* chain;       // [65536] deltas
    int next;              // nextToUpdate
};

struct HcOut {
    uint8_t* dst; int cap; int op; int ip; int anchor;
    SIMT_MEM void put(int at, uint32_t v) { if (at < cap) simt::stg_u8(dst + at, (uint8_t)v); }   // never outside [dst,dst+cap)
};

SIMT_DEV uint32_t hc_hash(const HcState& s, int p) { return (in32(s.src, p) * 2654435761u) >> 17; }   // :245-246

SIMT_DEV void hc_insert(HcState& s, int upto)                       // :358-373
{
    while (s.next < upto) {
        const int p = s.next;
        const uint32_t h = hc_hash(s, p);
        uint32_t delta = (uint32_t)p - s.heads[h];
        if (delta > 65535u) delta = 65535u;
        s.chain[p & 65535] = (uint16_t)delta;
        s.heads[h] = (uint32_t)p;
        s.next++;
    }
}

// equal bytes of src[a..] and src[b..] with a < limit as the stop (== the 8/4/2/1 scheme of :376-391)
SIMT_DEV int hc_common(const uint8_t* src, int a, int b, int limit)
{
    const int a0 = a;
    while (a + 4 <= limit) {
        const uint32_t x = in32(src, a) ^ in32(src, b);
        if (x) return a - a0 + ((simt::ffs(x) - 1) >> 3);
        a += 4; b += 4;
    }
    while (a < limit && simt::ldg_nc_u8(src + a) == simt::ldg_nc_u8(src + b)) { a++; b++; }
    return a - a0;
}

SIMT_DEV int hc_best(HcState& s, int ip, int matchlimit, int* mpos)  // :394-459 LZ4HC_InsertAndFindBestMatch
{
    const uint8_t* src = s.src;
    int attempts = 256, repl = 0, ml = 0;
    uint32_t delta = 0;
    hc_insert(s, ip);
    int ref = (int)s.heads[hc_hash(s, ip)];
    const uint32_t vip = in32(src, ip);
    if (ref >= ip - 4) {                                            // :411-420 repeat detector
        if (in32(src, ref) == vip) {
            delta = (uint32_t)(ip - ref) & 0xFFFFu;
            repl = ml = hc_common(src, ip + 4, ref + 4, matchlimit) + 4;
            *mpos = ref;
        }
        ref -= s.chain[ref & 65535];
    }
    while (ref >= ip - 65535 && attempts) {                         // :423-433
        attempts--;
        if (ref < 0) break;
        if (simt::ldg_nc_u8(src + ref + ml) == simt::ldg_nc_u8(src + ip + ml) && in32(src, ref) == vip) {
            const int mlt = hc_common(src, ip + 4, ref + 4, matchlimit) + 4;
            if (mlt > ml) { ml = mlt; *mpos = ref; }
        }
        ref -= s.chain[ref & 65535];
    }
    if (repl) {                                                     // :437-455
        int ptr = ip; const int end = ip + repl - 3;
        while (ptr < end - (int)delta) { s.chain[ptr & 65535] = (uint16_t)delta; ptr++; }
        do {
            s.chain[ptr & 65535] = (uint16_t)delta;
            s.heads[hc_hash(s, ptr)] = (uint32_t)ptr;
            ptr++;
        } while (ptr < end);
        s.next = end;
    }
    return ml;
}

SIMT_DEV int hc_wider(HcState& s, int ip, int start_limit, int matchlimit, int longest, int* mpos, int* spos)
{                                                                   // :462-518 LZ4HC_InsertAndGetWiderMatch
    const uint8_t* src = s.src;
    int attempts = 256;
    const int delta = ip - start_limit;
    hc_insert(s, ip);
    int ref = (int)s.heads[hc_hash(s, ip)];
    const uint32_t vip = in32(src, ip);
    while (ref >= ip - 65535 && attempts) {
        attempts--;
        if (ref < 0) break;
        if (simt::ldg_nc_u8(src + start_limit + longest) == simt::ldg_nc_u8(src + ref - delta + longest) &&
            in32(src, ref) == vip) {
            const int ipt = ip + 4 + hc_common(src, ip + 4, ref + 4, matchlimit);
            int st = ip, rt = ref;
            while (st > start_limit && rt > 0 && simt::ldg_nc_u8(src + st - 1) == simt::ldg_nc_u8(src + rt - 1)) { st--; rt--; }
            if (ipt - st > longest) { longest = ipt - st; *mpos = rt; *spos = st; }
        }
        ref -= s.chain[ref & 65535];
    }
    return longest;
}

SIMT_DEV int hc_put_len(HcOut& o, int at, int v)
{
    while (v > 254) { o.put(at++, 255); v -= 255; }
    o.put(at++, (uint32_t)v);
    return at;
}

SIMT_DEV bool hc_emit(const uint8_t* src, HcOut& o, int ml, int ref)  // :521-550 LZ4_encodeSequence; true = output full
{
    const int L = o.ip - o.anchor, tok = o.op++;
    uint32_t tv;
    if (o.op + L + 8 + (L >> 8) > o.cap) return true;                // :529
    if (L >= 15) { tv = 0xF0; o.op = hc_put_len(o, o.op, L - 15); } else tv = (uint32_t)L << 4;
    for (int i = 0; i < L; i++) o.put(o.op + i, simt::ldg_nc_u8(src + o.anchor + i));
    o.op += L;
    o.put(o.op, (uint32_t)(o.ip - ref) & 255); o.put(o.op + 1, ((uint32_t)(o.ip - ref) >> 8) & 255); o.op += 2;
    const int len = ml - 4;
    if (o.op + 6 + (L >> 8) > o.cap) return true;                    // :541 -- the LITERAL length, as the reference does
    if (len >= 15) { tv |= 15; o.op = hc_put_len(o, o.op, len - 15); } else tv |= (uint32_t)len;
    o.put(tok, tv);
    o.ip += ml; o.anchor = o.ip;
    return false;
}

// One block.  `state` = this thread's private HC_STATE_BYTES arena.  Returns bytes written, 0 = did not fit.
SIMT_DEV int hc_encode_block(void* state, const uint8_t* src, int n, uint8_t* dst, int cap)
{
    if (n < 0 || cap < 0) return 0;
    HcState s; s.src = src; s.heads = (uint32_t*)state; s.chain = (uint16_t*)((uint8_t*)state + 32768 * 4); s.next = 1;
    for (int i = 0; i < 32768 / 4; i++) simt::stg_v4(s.heads + 4 * i, uint4{0, 0, 0, 0});     // :330-337
    s.chain[0] = 0xFFFF;
    HcOut o{dst, cap, 0, 0, 0};
    const int mflimit = n - 12, matchlimit = n - 5;
    int ml, ml2, ml3, ml0, ref = 0, ref2 = 0, ref3 = 0, ref0, start2 = 0, start3 = 0, start0;

    o.ip = 1;                                                        // :581
    while (o.ip < mflimit) {                                         // :584
        ml = hc_best(s, o.ip, matchlimit, &ref);
        if (!ml) { o.ip++; continue; }
        start0 = o.ip; ref0 = ref; ml0 = ml;                         // :589-592
        bool to_search2 = true;
        for (;;) {
            if (to_search2) {                                        // _Search2  :594-622
                ml2 = (o.ip + ml < mflimit) ? hc_wider(s, o.ip + ml - 2, o.ip + 1, matchlimit, ml, &ref2, &start2) : ml;
                if (ml2 == ml) { if (hc_emit(src, o, ml, ref)) return 0; break; }
                if (start0 < o.ip && start2 < o.ip + ml0) { o.ip = start0; ref = ref0; ml = ml0; }
                if (start2 - o.ip < 3) { ml = ml2; o.ip = start2; ref = ref2; continue; }
            }
            // _Search3  :624-726
            if (start2 - o.ip < 18) {
                int new_ml = ml > 18 ? 18 : ml;
                if (o.ip + new_ml > start2 + ml2 - 4) new_ml = (start2 - o.ip) + ml2 - 4;
                const int corr = new_ml - (start2 - o.ip);
                if (corr > 0) { start2 += corr; ref2 += corr; ml2 -= corr; }
            }
            ml3 = (start2 + ml2 < mflimit) ? hc_wider(s, start2 + ml2 - 3, start2, matchlimit, ml2, &ref3, &start3) : ml2;
            if (ml3 == ml2) {                                        // :648-657 two sequences
                if (start2 < o.ip + ml) ml = start2 - o.ip;
                if (hc_emit(src, o, ml, ref)) return 0;
                o.ip = start2;
                if (hc_emit(src, o, ml2, ref2)) return 0;
                break;
            }
            if (start3 < o.ip + ml + 3) {                            // :659-691
                if (start3 >= o.ip + ml) {
                    if (start2 < o.ip + ml) {
                        const int corr = o.ip + ml - start2;
                        start2 += corr; ref2 += corr; ml2 -= corr;
                        if (ml2 < 4) { start2 = start3; ref2 = ref3; ml2 = ml3; }
                    }
                    if (hc_emit(src, o, ml, ref)) return 0;
                    o.ip = start3; ref = ref3; ml = ml3;
                    start0 = start2; ref0 = ref2; ml0 = ml2;
                    to_search2 = true; continue;
                }
                start2 = start3; ref2 = ref3; ml2 = ml3;
                to_search2 = false; continue;
            }
            if (start2 < o.ip + ml) {                                // :695-714
                if (start2 - o.ip < 15) {
                    if (ml > 18) ml = 18;
                    if (o.ip + ml > start2 + ml2 - 4) ml = (start2 - o.ip) + ml2 - 4;
                    const int corr = ml - (start2 - o.ip);
                    if (corr > 0) { start2 += corr; ref2 += corr; ml2 -= corr; }
                } else ml = start2 - o.ip;
            }
            if (hc_emit(src, o, ml, ref)) return 0;                  // :715
            o.ip = start2; ref = ref2; ml = ml2;
            start2 = start3; ref2 = ref3; ml2 = ml3;
            to_search2 = false;
        }
    }
    {                                                                // :729-739 last literals
        const int R = n - o.anchor;
        if ((uint32_t)(o.op + R + 1 + (R + 255 - 15) / 255) > (uint32_t)cap) return 0;
        if (R >= 15) { o.put(o.op++, 0xF0); o.op = hc_put_len(o, o.op, R - 15); } else o.put(o.op++, (uint32_t)R << 4);
        for (int i = 0; i < R; i++) o.put(o.op + i, simt::ldg_nc_u8(src + o.anchor + i));
        o.op += R;
    }
    return o.op;
}

}  // namespace lz4b200
