// lz4_lift.cuh -- how the stages of the asynchronous decode and Unwrap whose block offsets exist only on the device are
// staged out of page-locked host memory (capi.cu lz4b200_decode_batch_to_device_at_async,
// lz4b200_unwrap_batch_to_device_at_async).  The mirror image of lz4_land.cuh: it reads mapped host memory by 16-byte units.
//
// Block i of the batch spans [src_off[i], src_off[i+1]) of src, where src_off is what a packed asynchronous encode or Wrap
// has just written on the device.  The host knows each block's bound (a decode's compress_bound(dst_cap), an Unwrap
// packet's dst_cap + 8) but not its span, so a copy engine cannot be given the range to copy.  The host cuts the stages
// by bound and gives block i of a stage a slot at slot[i] of the staging buffer, slot[i+1] - slot[i] = the 16-aligned
// (bound + 32); slot[m] is the stage's size.  One kernel per stage then, from span[0..m] = src_off[b0..b1] and
// span[m+1] = src_off[n], both copied into device memory first so that no unit reads an offset over PCIe:
//   - entry i writes the decoder's entry: so[i] = slot[i] + (the host address of the span's first byte & 15), so that the
//     staged bytes keep their alignment mod 16, and sl[i] = the span; a rejected block gets the neutral entry (src_len 0,
//     dst_cap 0: lz4_wrap.cuh), which every decoder and the Unwrap prep pass over without reading or writing;
//   - unit u of the buffer (by binary search on slot[]) is unit k = u - slot[j] / 16 of block j's span: the aligned
//     16-byte unit of src that holds the span's first byte, plus 16 k.  It moves with one aligned load and one aligned
//     store, and only when it overlaps the span.
// A span is well-formed when 0 <= lo <= hi <= src_cap, hi - lo <= bound, and src_off[n] <= src_cap (otherwise the offload
// that wrote the offsets did not fit its destination, and which of its bytes landed is unknown).  Nothing of a rejected
// block is read; nothing outside [src, src + src_cap) is read, except the rest of an aligned unit that overlaps it.  After
// the decode, lift_status turns a rejected block's result into LZ4B200_E_ARG.
#pragma once
#include "simt.cuh"

namespace lz4b200 {

constexpr int32_t LIFT_E_ARG = -1;                                         // LZ4B200_E_ARG
constexpr int64_t LIFT_SLACK = 32;                                         // a slot's bytes beyond its bound

// The bytes of a slot for a block of `bound` bytes (host and device): the span, its offset in its first unit and at least
// 17 bytes of room behind it, which the decoders may read past a block's last byte.
constexpr int64_t lift_slot_bytes(int32_t bound) { return ((int64_t)bound + LIFT_SLACK + 15) & ~(int64_t)15; }

SIMT_DEV bool lift_ok(int64_t lo, int64_t hi, int64_t end, int64_t src_cap, int32_t bound)
{
    return end <= src_cap && 0 <= lo && lo <= hi && hi <= src_cap && hi - lo <= bound;
}

// Entry i of m.
SIMT_DEV void lift_entry(int32_t i, const uint8_t* src, int64_t src_cap, const int64_t* slot, const int64_t* span, int32_t m,
                         const int32_t* bound, int64_t* so, int32_t* sl, int32_t* dc)
{
    const int64_t lo = span[i], hi = span[i + 1];
    const bool ok = lift_ok(lo, hi, span[m + 1], src_cap, bound[i]);
    so[i] = slot[i] + (ok ? (int64_t)((uintptr_t)(src + lo) & 15) : 0);
    sl[i] = ok ? (int32_t)(hi - lo) : 0;
    if (!ok) dc[i] = 0;
}

// Unit u of the stage's staging buffer io (u < slot[m] / 16).
SIMT_DEV void lift_unit(int64_t u, const uint8_t* src, int64_t src_cap, const int64_t* slot, const int64_t* span, int32_t m,
                        const int32_t* bound, uint8_t* io)
{
    const int64_t at = 16 * u;
    int32_t j = 0, k = m;                                                  // slot[j] <= at < slot[k]
    while (k - j > 1) {
        const int32_t mid = (int32_t)(((int64_t)j + k) >> 1);
        if (slot[mid] <= at) j = mid; else k = mid;
    }
    const int64_t lo = span[j], hi = span[j + 1];
    if (lo == hi || !lift_ok(lo, hi, span[m + 1], src_cap, bound[j])) return;
    const uint8_t* first = src + lo;
    const uint8_t* p = first - ((uintptr_t)first & 15) + (at - slot[j]);
    if (p >= src + hi) return;
    simt::stg_v4(io + at, simt::ldg_nc_v4(p));
}

// Entry i of m, after the decode: a rejected block's result is LZ4B200_E_ARG.
SIMT_DEV void lift_status(int32_t i, int64_t src_cap, const int64_t* span, int32_t m, const int32_t* bound, int32_t* out)
{
    if (!lift_ok(span[i], span[i + 1], span[m + 1], src_cap, bound[i])) out[i] = LIFT_E_ARG;
}

}  // namespace lz4b200
