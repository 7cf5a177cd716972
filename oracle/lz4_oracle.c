/*
 * lz4_oracle.c -- TEST INFRASTRUCTURE ONLY.  Never shipped, never linked into lz4net_b200.
 *
 * An index-based, plain-C restatement of the LZ4 r93 block codec exactly as lz4net ships it
 * (lz4net generates its C# LZ4ps/LZ4pn codecs from, and compiles its LZ4mm/LZ4cc codecs out of,
 * original/lz4.c and original/lz4hc.c with LZ4_ARCH64=1 + LZ4_MK_OPT: src/adapters/cpp/lz4_64.h:5-9).
 * It exists so the GPU kernels have a byte-exact checker that travels to the GPU box.
 *
 * Parity pinning: tests/test_oracle.py proves this restatement byte-identical to the reference's own
 * sources compiled in place (oracle/_ref/liblz4net_ref.so, see Makefile) over thousands of seeded inputs,
 * all limited-output boundaries and the decoders' accept/reject decisions, and against the committed
 * golden vectors in tests/golden/ (generated from oracle/_ref by tests/golden/make_golden.py).
 *
 * Every function cites the reference lines it restates.  All reference citations are relative to
 * the root of a MiloszKrajewski/lz4net checkout.
 */
#include "lz4_oracle.h"
#include <string.h>
#include <stdlib.h>

enum {
    MINMATCH = 4,          /* original/lz4.c:182 */
    COPYLENGTH = 8,        /* :191 */
    LASTLITERALS = 5,      /* :192 */
    MFLIMIT = 12,          /* :193 */
    MINLENGTH = 13,        /* :194 */
    MAX_DISTANCE = 65535,  /* :197 */
    LZ4_64KLIMIT = 65547,  /* :565  (1<<16) + (MFLIMIT-1) */
    HC_ATTEMPTS = 256,     /* original/lz4hc.c:184 MAX_NB_ATTEMPTS */
    OPTIMAL_ML = 18        /* original/lz4hc.c:195 (ML_MASK-1)+MINMATCH */
};

static inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }

int lz4o_bound(int n) { return n + n / 255 + 16; }

/* length-extension bytes: a run of 255s then the remainder (0 allowed).
 * original/lz4.c:669-684 (literals) and :732 (matches: the 510/255 unrolling emits the same bytes). */
static inline int put_len_ext(uint8_t* dst, int op, int v)
{
    while (v > 254) { dst[op++] = 255; v -= 255; }
    dst[op++] = (uint8_t)v;
    return op;
}

/* ------------------------------------------------------------------------------------------------
 * Fast encoder.  original/lz4.c:573-771 (LZ4_compress64kCtx, n < 65547: 13-bit hash, u16 table,
 * no distance check) and :345-562 (LZ4_compressCtx: 12-bit hash, u32 table, MAX_DISTANCE checks).
 * Table entries are positions; the table is zero-filled so an empty bucket yields candidate 0 (:583,:651).
 * ---------------------------------------------------------------------------------------------- */
static int encode_fast(const uint8_t* src, int n, uint8_t* dst, int cap, int general)
{
    const int hshift = general ? 20 : 19;                 /* :185-187 vs :566-569 */
    const int mflimit = n - MFLIMIT;                      /* :361 / :590 */
    const int matchlimit = n - LASTLITERALS;              /* :366 / :596 */
    uint32_t* T = (uint32_t*)calloc(8192, sizeof(uint32_t));
    int ip = 0, anchor = 0, op = 0, ret = 0;
    if (!T) return 0;
#define HF(p) ((rd32(src + (p)) * 2654435761u) >> hshift)

    if (n < MINLENGTH) goto last_literals;                /* :387 / :615 */
    /* general variant inserts position 0 explicitly (:403) -- a no-op on a zeroed table */
    ip = 1;                                               /* :404 / :631 */
    for (;;) {
        int attempts = (1 << 6) + 3;                      /* :409 / :636 */
        int fwd = ip, ref, tok, L, M;
        for (;;) {                                        /* :415-429 / :642-654 */
            int step = attempts++ >> 6;
            uint32_t h;
            ip = fwd; fwd = ip + step;
            if (fwd > mflimit) goto last_literals;        /* bounds test precedes the probe */
            h = HF(ip);
            ref = (int)T[h]; T[h] = (uint32_t)ip;
            if (general && ref < ip - MAX_DISTANCE) continue;
            if (rd32(src + ref) == rd32(src + ip)) break;
        }
        while (ip > anchor && ref > 0 && src[ip - 1] == src[ref - 1]) { ip--; ref--; }   /* :432 / :657 */

        L = ip - anchor; tok = op++;
        if (op + L + (L >> 8) > cap - (2 + 1 + LASTLITERALS)) goto fail;                 /* :438 / :663 */
        if (L >= 15) { dst[tok] = 0xF0; op = put_len_ext(dst, op, L - 15); }
        else dst[tok] = (uint8_t)(L << 4);
        memcpy(dst + op, src + anchor, (size_t)L); op += L;                               /* :466 / :691 */

        for (;;) {                                                                        /* _next_match */
            uint32_t h;
            dst[op] = (uint8_t)(ip - ref); dst[op + 1] = (uint8_t)((ip - ref) >> 8); op += 2;  /* :470 / :695 */
            ip += MINMATCH; ref += MINMATCH; anchor = ip;
            while (ip < matchlimit && src[ref] == src[ip]) { ip++; ref++; }   /* == the 8/4/2/1 scheme :475-494 / :701-716 */
            M = ip - anchor;
            if (op + (M >> 8) > cap - (1 + LASTLITERALS)) goto fail;                      /* :501 / :728 */
            if (M >= 15) { dst[tok] += 15; op = put_len_ext(dst, op, M - 15); }
            else dst[tok] += (uint8_t)M;

            if (ip > mflimit) { anchor = ip; goto last_literals; }                        /* :516 / :736 */
            T[HF(ip - 2)] = (uint32_t)(ip - 2);                                           /* :519 / :739 */
            h = HF(ip); ref = (int)T[h]; T[h] = (uint32_t)ip;                             /* :523-525 / :743-745 */
            if ((!general || ref > ip - (MAX_DISTANCE + 1)) && rd32(src + ref) == rd32(src + ip)) {
                tok = op++; dst[tok] = 0; continue;                                       /* :531 / :751 */
            }
            break;
        }
        anchor = ip++;                                                                    /* :534 / :754 */
    }

last_literals: {
        int R = n - anchor;                                                               /* :540-551 / :760-767 */
        if (op + R + 1 + (R - 15 + 255) / 255 > cap) goto fail;
        if (R >= 15) { dst[op++] = 0xF0; op = put_len_ext(dst, op, R - 15); }
        else dst[op++] = (uint8_t)(R << 4);
        memcpy(dst + op, src + anchor, (size_t)R); op += R;
        ret = op;
    }
fail:
    free(T);
    return ret;
#undef HF
}

int lz4o_encode(const uint8_t* src, int n, uint8_t* dst, int cap)
{
    return encode_fast(src, n, dst, cap, n >= LZ4_64KLIMIT);   /* original/lz4.c:774-792 */
}

/* ------------------------------------------------------------------------------------------------
 * Decoders.  Accept/reject decisions follow the 64-bit flavour exactly; a rejected stream returns
 * -(input position) like the reference (the magnitude is unobservable through lz4net, whose wrappers
 * only test the sign: src/LZ4ps/LZ4Codec.Safe.cs:539-549).
 * One deliberate tightening: offset 0 is rejected (the reference would copy uninitialised output).
 * ---------------------------------------------------------------------------------------------- */
static inline void copy_match(uint8_t* dst, int op, int off, int len)
{
    /* overlap-aware forward byte copy == dec32/dec64-table + wild copy of original/lz4.c:869-909 */
    const uint8_t* s = dst + op - off; uint8_t* d = dst + op;
    for (int i = 0; i < len; i++) d[i] = s[i];
}

int lz4o_decode_known(const uint8_t* src, int isize, uint8_t* dst, int osize)   /* original/lz4.c:812-914 */
{
    int ip = 0, op = 0;
    const int bounded = isize >= 0;
#define NEED(k) do { if (bounded && ip + (k) > isize) return -ip - 1; } while (0)
    for (;;) {
        int token, L, M, off, end;
        NEED(1); token = src[ip++];
        L = token >> 4;
        if (L == 15) { int s; do { NEED(1); s = src[ip++]; L += s; if (L < 0) return -ip; } while (s == 255); }   /* :843 */
        end = op + L;
        if (end > osize - COPYLENGTH || end < op) {                      /* :847-857 */
            if (end != osize) return -ip;
            NEED(L); memcpy(dst + op, src + ip, (size_t)L); ip += L;
            return ip;                                                   /* bytes read */
        }
        NEED(L); memcpy(dst + op, src + ip, (size_t)L); ip += L; op = end;
        NEED(2); off = src[ip] | (src[ip + 1] << 8); ip += 2;            /* :862 */
        if (off > op || off == 0) return -ip;                            /* :863 */
        M = token & 15;
        if (M == 15) { int s; do { NEED(1); s = src[ip++]; M += s; if (M < 0) return -ip; } while (s == 255); }   /* :866 */
        end = op + M + MINMATCH;
        if (end > osize - LASTLITERALS || end < op) return -ip;          /* :893 last 5 bytes must be literals */
        copy_match(dst, op, off, M + MINMATCH); op = end;
    }
#undef NEED
}

int lz4o_decode_unknown(const uint8_t* src, int isize, uint8_t* dst, int max_out)   /* original/lz4.c:916-1044 */
{
    int ip = 0, op = 0;
    if (isize <= 0) return -1;                                           /* :949 (the reference returns -0) */
    for (;;) {
        int token, L, M, off, end;
        token = src[ip++];
        L = token >> 4;
        if (L == 15) { int s = 255; while (ip < isize && s == 255) { s = src[ip++]; L += s; if (L < 0) return -ip; } }   /* :959-963 */
        end = op + L;
        if (end > max_out - MFLIMIT || ip + L > isize - (2 + 1 + LASTLITERALS) || end < op) {       /* :968-978 */
            if (end > max_out || end < op) return -ip;
            if (ip + L != isize) return -ip;
            memcpy(dst + op, src + ip, (size_t)L); op += L;
            return op;                                                   /* bytes written */
        }
        memcpy(dst + op, src + ip, (size_t)L); ip += L; op = end;
        off = src[ip] | (src[ip + 1] << 8); ip += 2;                     /* :982 */
        if (off > op || off == 0) return -ip;                            /* :983 */
        M = token & 15;
        if (M == 15) {                                                   /* :986-999 */
            while (ip < isize - (LASTLITERALS + 1)) { int s = src[ip++]; M += s; if (M < 0) return -ip; if (s == 255) continue; break; }
        }
        end = op + M + MINMATCH;
        if (end > max_out - LASTLITERALS || end < op) return -ip;        /* :1025 */
        copy_match(dst, op, off, M + MINMATCH); op = end;
    }
}

/* ------------------------------------------------------------------------------------------------
 * LZ4HC.  original/lz4hc.c.  State (:231-237): heads[32768] u32 positions (zero-filled), chain[65536]
 * u16 deltas (0xFFFF-filled), next-to-update = 1 in the 64-bit flavour (:334).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    const uint8_t* src;
    uint32_t heads[32768];
    uint16_t chain[65536];
    int next;
} hc_t;

#define HH(s, p) ((rd32((s)->src + (p)) * 2654435761u) >> 17)            /* :245-246 HASH_LOG = 15 */

static void hc_insert(hc_t* s, int upto)                                  /* :358-373 LZ4HC_Insert */
{
    while (s->next < upto) {
        int p = s->next;
        uint32_t h = HH(s, p);
        size_t delta = (size_t)p - (size_t)s->heads[h];
        if (delta > MAX_DISTANCE) delta = MAX_DISTANCE;
        s->chain[p & 65535] = (uint16_t)delta;
        s->heads[h] = (uint32_t)p;
        s->next++;
    }
}

static int hc_common(const uint8_t* src, int a, int b, int limit)         /* :376-391 LZ4HC_CommonLength */
{
    int a0 = a;
    while (a < limit && src[b] == src[a]) { a++; b++; }
    return a - a0;
}

static int hc_best(hc_t* s, int ip, int matchlimit, int* mpos)            /* :394-459 LZ4HC_InsertAndFindBestMatch */
{
    const uint8_t* src = s->src;
    int attempts = HC_ATTEMPTS, repl = 0, ml = 0, ref;
    uint16_t delta = 0;
    hc_insert(s, ip);
    ref = (int)s->heads[HH(s, ip)];
    if (ref >= ip - 4) {                                                  /* :411-420 repeat detector */
        if (rd32(src + ref) == rd32(src + ip)) {
            delta = (uint16_t)(ip - ref);
            repl = ml = hc_common(src, ip + MINMATCH, ref + MINMATCH, matchlimit) + MINMATCH;
            *mpos = ref;
        }
        ref -= s->chain[ref & 65535];                                     /* no attempt spent */
    }
    while (ref >= ip - MAX_DISTANCE && attempts) {                        /* :423-433 */
        attempts--;
        if (ref < 0) break;                                               /* defensive; unreachable for sane state */
        if (src[ref + ml] == src[ip + ml] && rd32(src + ref) == rd32(src + ip)) {
            int mlt = hc_common(src, ip + MINMATCH, ref + MINMATCH, matchlimit) + MINMATCH;
            if (mlt > ml) { ml = mlt; *mpos = ref; }
        }
        ref -= s->chain[ref & 65535];
    }
    if (repl) {                                                           /* :437-455 complete the table for the run */
        int ptr = ip, end = ip + repl - (MINMATCH - 1);
        while (ptr < end - (int)delta) { s->chain[ptr & 65535] = delta; ptr++; }
        do {
            s->chain[ptr & 65535] = delta;
            s->heads[HH(s, ptr)] = (uint32_t)ptr;
            ptr++;
        } while (ptr < end);
        s->next = end;
    }
    return ml;
}

static int hc_wider(hc_t* s, int ip, int start_limit, int matchlimit, int longest, int* mpos, int* spos)
{                                                                         /* :462-518 LZ4HC_InsertAndGetWiderMatch */
    const uint8_t* src = s->src;
    int attempts = HC_ATTEMPTS, ref;
    const int delta = ip - start_limit;
    hc_insert(s, ip);
    ref = (int)s->heads[HH(s, ip)];
    while (ref >= ip - MAX_DISTANCE && attempts) {
        attempts--;
        if (ref < 0) break;
        if (src[start_limit + longest] == src[ref - delta + longest] && rd32(src + ref) == rd32(src + ip)) {
            int ipt = ip + MINMATCH + hc_common(src, ip + MINMATCH, ref + MINMATCH, matchlimit);
            int st = ip, rt = ref;
            while (st > start_limit && rt > 0 && src[st - 1] == src[rt - 1]) { st--; rt--; }   /* :505 */
            if (ipt - st > longest) { longest = ipt - st; *mpos = rt; *spos = st; }
        }
        ref -= s->chain[ref & 65535];
    }
    return longest;
}

typedef struct { uint8_t* dst; int cap; int op; int ip; int anchor; } hc_out_t;

static int hc_emit(const uint8_t* src, hc_out_t* o, int ml, int ref)      /* :521-550 LZ4_encodeSequence */
{
    int L = o->ip - o->anchor, tok = o->op++, len;
    if (o->op + L + (2 + 1 + LASTLITERALS) + (L >> 8) > o->cap) return 1;         /* :529 */
    if (L >= 15) { o->dst[tok] = 0xF0; o->op = put_len_ext(o->dst, o->op, L - 15); }
    else o->dst[tok] = (uint8_t)(L << 4);
    memcpy(o->dst + o->op, src + o->anchor, (size_t)L); o->op += L;
    o->dst[o->op] = (uint8_t)(o->ip - ref); o->dst[o->op + 1] = (uint8_t)((o->ip - ref) >> 8); o->op += 2;
    len = ml - MINMATCH;
    if (o->op + (1 + LASTLITERALS) + (L >> 8) > o->cap) return 1;                 /* :541 uses the LITERAL length (normative) */
    if (len >= 15) { o->dst[tok] += 15; o->op = put_len_ext(o->dst, o->op, len - 15); }
    else o->dst[tok] += (uint8_t)len;
    o->ip += ml; o->anchor = o->ip;
    return 0;
}

int lz4o_encode_hc(const uint8_t* src, int n, uint8_t* dst, int cap)      /* :557-755 */
{
    hc_t* s = (hc_t*)malloc(sizeof(hc_t));
    hc_out_t o = { dst, cap, 0, 0, 0 };
    const int mflimit = n - MFLIMIT, matchlimit = n - LASTLITERALS;
    int ml, ml2, ml3, ml0, ref = 0, ref2 = 0, ref3 = 0, ref0, start2 = 0, start3 = 0, start0, ret = 0;
    if (!s) return 0;
    s->src = src; s->next = 1;                                            /* :330-337 (64-bit: base+1) */
    memset(s->heads, 0, sizeof s->heads);
    memset(s->chain, 0xFF, sizeof s->chain);

    o.ip = 1;                                                             /* :581 */
    while (o.ip < mflimit) {                                              /* :584 */
        ml = hc_best(s, o.ip, matchlimit, &ref);
        if (!ml) { o.ip++; continue; }
        start0 = o.ip; ref0 = ref; ml0 = ml;                              /* :589-592 */
search2:
        if (o.ip + ml < mflimit) ml2 = hc_wider(s, o.ip + ml - 2, o.ip + 1, matchlimit, ml, &ref2, &start2);   /* :595-597 */
        else ml2 = ml;
        if (ml2 == ml) { if (hc_emit(src, &o, ml, ref)) goto fail; continue; }    /* :599-603 */
        if (start0 < o.ip && start2 < o.ip + ml0) { o.ip = start0; ref = ref0; ml = ml0; }   /* :605-613 */
        if (start2 - o.ip < 3) { ml = ml2; o.ip = start2; ref = ref2; goto search2; }        /* :616-622 */
search3:
        if (start2 - o.ip < OPTIMAL_ML) {                                 /* :628-641 */
            int new_ml = ml, corr;
            if (new_ml > OPTIMAL_ML) new_ml = OPTIMAL_ML;
            if (o.ip + new_ml > start2 + ml2 - MINMATCH) new_ml = (start2 - o.ip) + ml2 - MINMATCH;
            corr = new_ml - (start2 - o.ip);
            if (corr > 0) { start2 += corr; ref2 += corr; ml2 -= corr; }
        }
        if (start2 + ml2 < mflimit) ml3 = hc_wider(s, start2 + ml2 - 3, start2, matchlimit, ml2, &ref3, &start3);   /* :644-646 */
        else ml3 = ml2;
        if (ml3 == ml2) {                                                 /* :648-657 two sequences */
            if (start2 < o.ip + ml) ml = start2 - o.ip;
            if (hc_emit(src, &o, ml, ref)) goto fail;
            o.ip = start2;
            if (hc_emit(src, &o, ml2, ref2)) goto fail;
            continue;
        }
        if (start3 < o.ip + ml + 3) {                                     /* :659-691 no room for match 2 */
            if (start3 >= o.ip + ml) {
                if (start2 < o.ip + ml) {
                    int corr = o.ip + ml - start2;
                    start2 += corr; ref2 += corr; ml2 -= corr;
                    if (ml2 < MINMATCH) { start2 = start3; ref2 = ref3; ml2 = ml3; }
                }
                if (hc_emit(src, &o, ml, ref)) goto fail;
                o.ip = start3; ref = ref3; ml = ml3;
                start0 = start2; ref0 = ref2; ml0 = ml2;
                goto search2;
            }
            start2 = start3; ref2 = ref3; ml2 = ml3;
            goto search3;
        }
        if (start2 < o.ip + ml) {                                         /* :695-714 three ascending matches */
            if (start2 - o.ip < 15) {
                int corr;
                if (ml > OPTIMAL_ML) ml = OPTIMAL_ML;
                if (o.ip + ml > start2 + ml2 - MINMATCH) ml = (start2 - o.ip) + ml2 - MINMATCH;
                corr = ml - (start2 - o.ip);
                if (corr > 0) { start2 += corr; ref2 += corr; ml2 -= corr; }
            } else ml = start2 - o.ip;
        }
        if (hc_emit(src, &o, ml, ref)) goto fail;                         /* :715 */
        o.ip = start2; ref = ref2; ml = ml2;                              /* :717-723 */
        start2 = start3; ref2 = ref3; ml2 = ml3;
        goto search3;
    }
    {                                                                     /* :729-739 last literals */
        int R = n - o.anchor;
        if ((unsigned)(o.op + R + 1 + (R + 255 - 15) / 255) > (unsigned)cap) goto fail;
        if (R >= 15) { dst[o.op++] = 0xF0; o.op = put_len_ext(dst, o.op, R - 15); }
        else dst[o.op++] = (uint8_t)(R << 4);
        memcpy(dst + o.op, src + o.anchor, (size_t)R); o.op += R;
        ret = o.op;
    }
fail:
    free(s);
    return ret;
}

/* LZ4_uncompress-shaped (3-argument, unbounded reads) wrapper so oracle_mt.c can time the port decoder too */
int lz4o_decode3(const char* src, char* dst, int osize)
{
    return lz4o_decode_known((const uint8_t*)src, -1, (uint8_t*)dst, osize);
}

/* LZ4_compress[HC]_limitedOutput-shaped wrappers (src, dst, isize, cap) for oracle_mt.c: the port's own argument
 * order is (src, isize, dst, cap) */
int lz4o_encode4(const char* src, char* dst, int isize, int cap) { return lz4o_encode((const uint8_t*)src, isize, (uint8_t*)dst, cap); }
int lz4o_encode_hc4(const char* src, char* dst, int isize, int cap) { return lz4o_encode_hc((const uint8_t*)src, isize, (uint8_t*)dst, cap); }
