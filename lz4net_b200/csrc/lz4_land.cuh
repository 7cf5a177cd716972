// lz4_land.cuh -- where the stages of the asynchronous packed encode into page-locked host memory land (capi.cu
// lz4b200_encode_batch_packed_from_device_async).
//
// A stage's encoder has written its blocks into dense device slots (block i at dof[i], len[i] bytes) and the scan has
// produced the stage-local offsets (off[0..m]: the exclusive prefix sum of max(len, 0), off[m] the stage's total).  Its
// place in the caller's destination is known only on the device: it starts at the running total the previous stage left
// (base; the carry cells of lz4_packed.cuh).  One kernel per stage writes the absolute offsets, the lengths and the new
// running total, and, when everything up to the stage's end fits total_cap, moves the stage's bytes into the destination
// through its device (mapped) address.
//
// The bytes move gathered by OUTPUT: unit u is the 16-byte-aligned unit u of the destination range [dst + base,
// dst + base + off[m]), counted from the aligned unit that holds its first byte.  The thread that owns a unit finds the
// block holding its first byte by binary search on off[], assembles the unit from the dense slots and stores it with one
// 16-byte store -- a warp writes 512 contiguous aligned bytes, whole lines over PCIe -- or, for a unit the range covers
// only in part (its head and its tail), with byte stores of exactly the covered bytes.  Adjacent stages therefore share at
// most one unit and never write each other's bytes of it, so the order between them does not matter.  Nothing outside
// [dst + base, dst + base + off[m]) is written, and a stage that does not fit writes no byte of dst at all.
//
// The dense slots are read with aligned 16-byte loads up to 31 bytes past a block's bytes: the slot buffer holds 64
// bytes behind its last slot.
#pragma once
#include "simt.cuh"
#include "lz4_copy.cuh"

namespace lz4b200 {

// The stage's units of 16 bytes (0 for an empty stage).
SIMT_DEV int64_t land_units(const uint8_t* at, int64_t total)
{
    return total > 0 ? ((int64_t)((uintptr_t)at & 15) + total + 15) >> 4 : 0;
}

// Entry i of the stage's results, thread i of m + 1: out_off[i] = base + off[i] (out_off[m] = the new running total, which
// the next stage writes again as its out_off[0]), out_len[i] = len[i]; thread m also leaves the running total for the
// next stage in *total_out.  A null out_off or out_len is not written (an LZ4Stream encode keeps only the total).
SIMT_DEV void land_place(int64_t i, const int32_t* len, const int64_t* off, int32_t m, int64_t base, int64_t* out_off,
                         int32_t* out_len, int64_t* total_out)
{
    if (i > m) return;
    if (out_off) out_off[i] = base + off[i];
    if (i == m) *total_out = base + off[m];
    else if (out_len) out_len[i] = len[i];
}

// Unit u of the stage's bytes at `at` (= dst + base).
SIMT_DEV void land_unit(int64_t u, const uint8_t* dense, const int64_t* dof, const int64_t* off, int32_t m, uint8_t* at)
{
    const int64_t total = off[m];
    const int64_t u_lo = 16 * u - (int64_t)((uintptr_t)at & 15);          // the unit's first byte, stage-relative
    const int64_t lo = u_lo > 0 ? u_lo : 0, hi = u_lo + 16 < total ? u_lo + 16 : total;
    if (lo >= hi) return;
    int32_t j = 0, k = m;                                                 // off[j] <= lo < off[k]
    while (k - j > 1) {
        const int32_t mid = (int32_t)(((int64_t)j + k) >> 1);
        if (off[mid] <= lo) j = mid; else k = mid;
    }
    uint8_t* d = at + u_lo;
    const bool whole = hi - lo == 16;
    if (whole && hi <= off[j + 1]) {
        // one block covers the unit: the two aligned words around its bytes, shifted
        const uint8_t* s = dense + dof[j] + (lo - off[j]);
        const uint32_t r = (uint32_t)((uintptr_t)s & 15);
        const uint8_t* sa = s - r;
        const uint4 w = simt::ldg_nc_v4(sa);
        simt::stg_v4(d, r ? shift16(w, simt::ldg_nc_v4(sa + 16), r) : w);
        return;
    }
    uint64_t x0 = 0, x1 = 0;
    for (int64_t p = lo; p < hi; p++) {
        while (p >= off[j + 1]) j++;                                      // (blocks of 0 bytes are passed over)
        const uint32_t b = simt::ldg_nc_u8(dense + dof[j] + (p - off[j]));
        const int q = (int)(p - u_lo);
        if (!whole) simt::stg_u8(d + q, (uint8_t)b);
        else if (q < 8) x0 |= (uint64_t)b << (8 * q);
        else x1 |= (uint64_t)b << (8 * (q - 8));
    }
    if (whole) {
        uint4 v;
        v.x = (uint32_t)x0; v.y = (uint32_t)(x0 >> 32); v.z = (uint32_t)x1; v.w = (uint32_t)(x1 >> 32);
        simt::stg_v4(d, v);
    }
}

}  // namespace lz4b200
