// lz4_measure.cuh -- the decoded size of a compressed block without decoding it: ONE LANE per block, headers only.
//
// Every accept / reject decision of the decoders (lz4_decode.cuh decode_careful, lz4_decode_lpb.cuh) depends on the
// stream's STRUCTURE alone -- tokens, length bytes, offsets, the input and output positions -- never on the contents of a
// literal run or a match (oracle/lz4_oracle.c:138-193).  A walk over the headers that skips the payload therefore
// predicts the decoder's result exactly without writing a byte:
//   unknown size (KNOWN = false): the bytes the decoder would write, or a negative value;
//   known size   (KNOWN = true):  the bytes the decoder would read,  or a negative value.
// Non-negative results equal the decoders'; negative ones agree in sign only (the magnitude is not part of the contract,
// DESIGN §5).  The rules below restate decode_careful / the lpb decoder's general path one by one, the 64-bit flavour's
// with the `end < op` overflow guards (as length limits) and offset 0 rejected.
//
// Input: aligned 16-byte loads through the read-only path; the lane keeps the unit it read last in four registers, so a
// header costs one load when it lies in a fresh unit and none otherwise.  Literal runs and matches are skipped by moving
// the cursor; runs of 255 length bytes (a 64 KiB literal run has ~257 of them) are counted a unit at a time.  Every read
// lies in a 16-byte unit that holds a stream byte: nothing outside [src, src + isize) rounded out to 16 bytes is touched,
// whatever the stream contains.
#pragma once
#include "simt.cuh"

namespace lz4b200 {

struct MeasureInput {
    const uint8_t* abase;              // stream rounded down to 16 bytes
    uint32_t skew;                     // src - abase
    uint32_t unit = 0xFFFFFFFFu;       // aligned offset (from abase) of the unit held in w
    uint32_t w[4] = {0, 0, 0, 0};

    SIMT_MEM void load(uint32_t p)     // make the unit holding stream byte p current
    {
        const uint32_t u = (p + skew) & ~15u;
        if (u != unit) {
            const uint4 v = simt::ldg_nc_v4(abase + u);
            w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w; unit = u;
        }
    }
    SIMT_MEM uint32_t word(uint32_t o) const { return o < 8 ? (o < 4 ? w[0] : w[1]) : (o < 12 ? w[2] : w[3]); }
    SIMT_MEM uint32_t byte(uint32_t p)
    {
        load(p);
        const uint32_t o = (p + skew) & 15u;
        return (word(o) >> (8u * (o & 3u))) & 255u;
    }
    // bytes of value 255 from stream position p up to the end of p's unit (load(p) first)
    SIMT_MEM uint32_t ff_run(uint32_t p) const
    {
        const uint32_t o = (p + skew) & 15u;
        const uint64_t lo = ~((uint64_t)w[1] << 32 | w[0]), hi = ~((uint64_t)w[3] << 32 | w[2]);   // non-zero bytes: not 255
        auto first_set_byte = [](uint64_t v) -> uint32_t {
            const uint32_t l = (uint32_t)v;
            return (uint32_t)(l ? simt::ffs(l) - 1 : 31 + simt::ffs((uint32_t)(v >> 32))) >> 3;
        };
        uint32_t end = 16;                                          // index of the first non-255 byte at or after o
        if (o < 8) {
            const uint64_t m = lo >> (8u * o);
            end = m ? o + first_set_byte(m) : (hi ? 8u + first_set_byte(hi) : 16u);
        } else {
            const uint64_t m = hi >> (8u * (o - 8u));
            end = m ? o + first_set_byte(m) : 16u;
        }
        return end - o;
    }
};

// The extension bytes of a literal or match length, starting at q with the value v: every byte is read only while
// q < qlim and v <= LIM, a byte other than 255 ends the length.  strict (the known-size decoder): a byte that may not be
// read makes the stream malformed (-1); otherwise the length simply ends there and the caller's checks decide.
SIMT_DEV int measure_ext(MeasureInput& in, int& q, int v, int qlim, bool strict)
{
    constexpr int LIM = 0x3FFFFFFF;
    for (;;) {
        if (q >= qlim || v > LIM) return strict ? -1 : v;
        in.load((uint32_t)q);
        int k = (int)in.ff_run((uint32_t)q);
        if (k == 0) { v += (int)in.byte((uint32_t)q); q++; return v; }
        // k bytes of 255 in a row: each of them would be read (and continue the length) while the limits hold
        if (k > qlim - q) k = qlim - q;
        const int klim = (LIM - v) / 255 + 1;
        if (k > klim) k = klim;
        v += 255 * k; q += k;
    }
}

template <bool KNOWN>
SIMT_DEV int measure_block(const uint8_t* src, int isize, int cap)
{
    constexpr int LIM = 0x3FFFFFFF;
    if (isize <= 0 || cap < 0) return -1;                         // original/lz4.c:949; a block has >= 1 token
    MeasureInput in;
    in.skew = (uint32_t)((uintptr_t)src & 15); in.abase = src - in.skew;
    int ip = 0, op = 0;
    for (;;) {
        // ---- token + literals (:843-857 / :959-978) ----
        if (ip >= isize) return -ip - 1;
        const uint32_t token = in.byte((uint32_t)ip); ip++;
        int L = (int)(token >> 4);
        if (L == 15) {
            L = measure_ext(in, ip, L, isize, KNOWN);
            if (L < 0 || L > LIM) return -ip - 1;
        }
        if (L > isize - ip || L > cap - op) return -ip - 1;
        const int end = op + L;
        const bool last = KNOWN ? end > cap - 8 : (end > cap - 12 || ip + L > isize - 8);
        const bool ok = last ? (KNOWN ? (end == cap && ip + L <= isize) : (end <= cap && ip + L == isize)) : ip + L + 2 <= isize;
        if (!ok) return -ip - 1;
        ip += L; op = end;
        if (last) return KNOWN ? ip : op;
        // ---- offset + match (:862-893 / :982-1025) ----
        const uint32_t off = in.byte((uint32_t)ip) | (in.byte((uint32_t)ip + 1) << 8);
        ip += 2;
        if (off == 0 || off > (uint32_t)op) return -ip - 1;       // offset 0 rejected by design
        int M = (int)(token & 15);
        if (M == 15) {
            M = measure_ext(in, ip, M, KNOWN ? isize : isize - 6, KNOWN);
            if (M < 0 || M > LIM) return -ip - 1;
        }
        if (M > cap - op || op + M + 4 > cap - 5) return -ip - 1; // the last 5 bytes are literals
        op += M + 4;
    }
}

}  // namespace lz4b200
