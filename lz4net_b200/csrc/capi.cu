// capi.cu -- the C ABI of liblz4b200.so (include/lz4b200.h): context, batched entry points, single-block entry points.
//
// Every call on host memory (the batches with LZ4B200_MEM_HOST, the packed encode, the measure pass, the single-block entry
// points, and the LZ4Stream and Wrap / Unwrap calls) goes through one software pipeline, run_host: the block list is cut
// into chunks, and for each chunk H2D(inputs) -> kernel -> D2H(outputs) is enqueued on one of NSLOT streams, so that the
// copy engines (both PCIe directions) and the SMs work on different chunks at the same time.  The mixed-memory batches
// (MEM_DEVICE_TO_HOST, MEM_HOST_TO_DEVICE and the packed encode from device memory) and the LZ4Stream and Wrap / Unwrap
// calls between device and host memory go through it too, skipping the copy of whichever side is already on the device;
// so does the packed unknown-size decode from host into device memory, whose output offset is carried across the stages
// on the device (lz4_packed.cuh).  What a stage runs is named by its caller (Stage); the codec operation by Op.
// The LZ4Stream frames and the Wrap headers are written on the device (lz4_stream.cuh, lz4_wrap.cuh) whichever side the
// caller's bytes are on; the host only reads headers (framing.cpp).  There is no CPU codec in this library: if the device
// or the kernel image is unusable every entry point reports an error.
#include "../../include/lz4b200.h"
#include "framing.h"
#include "kernels.h"
#include "lz4_packed.cuh"
#include "lz4_stream.cuh"
#include "lz4_wrap.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

using namespace lz4b200;

namespace {

thread_local std::string g_err = "";

int fail(int code, const std::string& msg) { g_err = msg; return code; }
int cuda_fail(cudaError_t e, const char* what)
{
    g_err = std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")";
    return LZ4B200_E_CUDA;
}
#define CU(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return cuda_fail(e_, #x); } while (0)

constexpr int NSLOT = 3;                       // pipeline depth of host-memory batches
constexpr int NCOUNTER = 256;
constexpr size_t HOST_CHUNK_BYTES_DEFAULT = 128u << 20; // src + dst bytes per pipeline stage (on H100 the best of 32..512 MiB: profiles/README.md)

// Grow-only buffers that free themselves (the context's device is current when a context is destroyed): device memory,
// grown with an eighth to spare, or page-locked host memory.
template <bool PINNED>
struct Buf {
    void* p = nullptr; size_t cap = 0;
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    ~Buf() { release(); }
    cudaError_t reserve(size_t n)
    {
        if (n <= cap) return cudaSuccess;
        release();
        const size_t want = PINNED ? n + 4096 : n + (n >> 3) + 4096;
        cudaError_t e = PINNED ? cudaMallocHost(&p, want) : cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) (PINNED ? cudaFreeHost(p) : cudaFree(p)); p = nullptr; cap = 0; }
};
using DevBuf = Buf<false>;
using PinBuf = Buf<true>;

// Pageable host memory (a managed caller's `fixed` byte[]): cudaMemcpyAsync from / to it is staged by the driver through
// its own small pinned buffers, synchronously (several times slower than from pinned memory).  The library
// stages such buffers itself, a pipeline chunk at a time, with a handful of host threads doing the memcpy into / out of
// its pinned chunk buffers while the previous chunks are on the wire.
constexpr int STAGE_THREADS = 8;
constexpr size_t STAGE_PARALLEL_MIN = 4u << 20;

void par_ranges(size_t n, size_t min_parallel, const std::function<void(size_t, size_t)>& fn)
{
    if (n < min_parallel) { fn(0, n); return; }
    std::vector<std::thread> th;
    const size_t per = (n + STAGE_THREADS - 1) / STAGE_THREADS;
    for (int t = 1; t < STAGE_THREADS; t++) {
        const size_t lo = per * t, hi = std::min(n, lo + per);
        if (lo < hi) th.emplace_back(fn, lo, hi);
    }
    fn(0, std::min(n, per));
    for (auto& t : th) t.join();
}
void par_memcpy(void* dst, const void* src, size_t n)
{
    par_ranges(n, STAGE_PARALLEL_MIN, [&](size_t lo, size_t hi) { std::memcpy((uint8_t*)dst + lo, (const uint8_t*)src + lo, hi - lo); });
}
bool is_pageable(const void* p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}

struct Slot {
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    cudaEvent_t carried = nullptr;         // the packed decode into device memory: the stage's placement step is enqueued
    DevBuf src, dst, meta, packed, offs, scan;
    PinBuf hmeta, hsrc, hout;              // pinned: chunk metadata, staged pageable sources, staged outputs
};

// One chunk's metadata, laid out the same in the slot's hmeta (host) and meta (device, which has no packed_off):
// int64 src_off[m] | int64 dst_off[m] | int32 src_len[m] | int32 dst_cap[m] | int32 aux[m] | int32 out_len[m] |
// int64 packed_off[m+1].  aux is used by the LZ4Stream and Unwrap calls only: the frame sizes of an encode (written on the
// device), the stored payload lengths of a decode (copied up with the first four arrays).  A Wrap encode keeps the codec's
// view of its packets (WrapScratch) in the device block behind out, at WRAP_META_OFFSET * m bytes: the slots are in flight
// at once, so it is theirs.  The packed decode into device memory keeps its stage's "fits" flag (an int) in the same
// place, for the same reason.
struct Meta {
    int64_t *so, *dof; int32_t *sl, *dc, *aux, *out; int64_t* off;
    Meta(void* p, int32_t m) : so((int64_t*)p), dof(so + m), sl((int32_t*)(dof + m)), dc(sl + m), aux(dc + m), out(aux + m),
                               off((int64_t*)(((uintptr_t)(out + m) + 7) & ~(uintptr_t)7)) {}
};
// The codec's view of n packets (int64 off[n] | int32 len[n] | int32 cap[n] | int32 res[n]) at p.
constexpr size_t WRAP_SCRATCH_BYTES = sizeof(int64_t) + 3 * sizeof(int32_t);
WrapScratch wrap_scratch_at(void* p, int32_t n)
{
    int32_t* len = (int32_t*)((int64_t*)p + n);
    return WrapScratch{(int64_t*)p, len, len + n, len + 2 * n};
}
constexpr size_t META_BYTES = 32, WRAP_META_OFFSET = 32, WRAP_META_BYTES = WRAP_META_OFFSET + WRAP_SCRATCH_BYTES;

// The operations of the batch codec.
enum class Op { ENCODE_FAST, ENCODE_HC, DECODE_KNOWN, DECODE_UNKNOWN, MEASURE_KNOWN, MEASURE_UNKNOWN };
constexpr Op encode_op(bool hc) { return hc ? Op::ENCODE_HC : Op::ENCODE_FAST; }
constexpr bool is_encode(Op op) { return op == Op::ENCODE_FAST || op == Op::ENCODE_HC; }
constexpr bool is_decode(Op op) { return op == Op::DECODE_KNOWN || op == Op::DECODE_UNKNOWN; }
constexpr bool is_measure(Op op) { return op == Op::MEASURE_KNOWN || op == Op::MEASURE_UNKNOWN; }

// What a stage of the host pipeline (run_host) runs on its chunk.
enum class Stage {
    CODEC,            // the operation (run_device)
    STREAM_ENCODE,    // the encode, then the chunks' LZ4Stream frames (lz4_stream.cuh) in place of the compaction: APPEND
                      // lands the frames, out_off[i] = where frame i starts
    WRAP_ENCODE,      // prep -> the encode -> finish (run_wrap, lz4_wrap.cuh): dst_cap[i] = the packet's capacity,
                      // src_len[i] + 8; the slot then holds whole packets, which land like the blocks of an encode
    FRAMED_DECODE,    // the known-size decode of LZ4Stream chunks or Unwrap packets: stored[i] != 0 marks a stored one, whose
                      // payload the stored-copy step copies while the decoder gets the neutral entry (src_len 0, dst_cap 0);
                      // in host memory it lands like a decoded block of dst_cap[i] bytes
    PLACED_DECODE,    // the packed unknown-size decode into device memory, its output offset carried across the stages
};

}  // namespace

struct lz4b200_ctx {
    int device = 0;
    DeviceInfo dev{};
    uint32_t* counters = nullptr;
    int next_counter = 0;
    DevBuf hc_arena, compact_tmp;
    DevBuf packed_caps;                    // lz4b200_decode_batch_packed: per-block capacities + the "fits" flag (serialised like compact_tmp)
    DevBuf wrap_tmp;                       // the device Wrap / Unwrap calls: the codec's view of the packets (serialised like compact_tmp)
    cudaEvent_t hc_done = nullptr;         // the HC state arena is shared: HC launches are chained through this event
    cudaEvent_t compact_done = nullptr;    // likewise compact_tmp, packed_caps and wrap_tmp (call_scratch)
    cudaEvent_t entry = nullptr;           // mixed-memory batches: recorded on the caller's stream, waited on by every slot
    int64_t* carry = nullptr;              // the packed decode into device memory: NSLOT cells, the running output offset behind each slot's stage
    int decode_lanes = 16;                 // lanes per block for device-memory batches (+100 = output-staged variant)
    bool decode_lanes_auto = true;         // host-memory batches: chosen per chunk from the compression ratio
    int encode_ctas_per_sm = 0;            // encoder warps (= blocks in flight) per SM: 0 = as many as shared memory holds tables for (14)
    int encode_variant = 2;                // same-hash detection inside a round: 1 exact votes, 2 optimistic (default)
    int encode_tune[4] = {512, 12, 8, 24}; // prefetch distance, lane_copy_max, probe_max, wide_min (lz4_encode.cuh EncTune)
    size_t host_chunk_bytes = HOST_CHUNK_BYTES_DEFAULT;
    int hc_concurrency = 131072;         // blocks in flight (one thread each, 256 KiB state: 32 GiB of arena at this default)
    int hc_kernel = -1;                  // -1: chosen per batch (encode.cu launch_encode_hc_auto); 0: one thread per block (any block size); one warp per block (on a static index for blocks <= 64 KiB, over a sliding 64 KiB window above; what neither describes goes to 0): 1 = block <= 64 KiB staged in shared memory, 2 = nothing in shared memory
    int hc_warps_per_sm = 0;             // warp kernels: blocks in flight per SM (0 = 3 for kernel 1, 32 for kernel 2)
    Slot slot[NSLOT];
    int64_t launches = 0;
    std::mutex mu;

    uint32_t* counter() { uint32_t* c = counters + next_counter; next_counter = (next_counter + 4) % NCOUNTER; return c; }   // fours: [block counter, decoder pick, two more counters]
    int pinned_lanes() const { return decode_lanes_auto ? 0 : decode_lanes; }   // 0: the decoder is picked on the device
};

namespace {

struct DeviceGuard {
    int prev = -1; bool ok;
    explicit DeviceGuard(int dev) { ok = cudaGetDevice(&prev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// The context's lock and its device for the rest of a call; rc = LZ4B200_E_CUDA when the device could not be made current.
struct CallGuard {
    std::lock_guard<std::mutex> lock;
    DeviceGuard dev;
    int rc;
    explicit CallGuard(lz4b200_ctx* c)
        : lock(c->mu), dev(c->device), rc(dev.ok ? LZ4B200_OK : fail(LZ4B200_E_CUDA, "cudaSetDevice failed")) {}
};

// The context's call scratch (compact_tmp, packed_caps, wrap_tmp) is shared by the device calls on every stream.  A call
// grows the buffers it needs to at least these sizes -- behind one cudaDeviceSynchronize, since an earlier call may still
// be using them -- and orders `st` behind the last call that used them.  The caller records compact_done on `st` once its
// launches are in.
int call_scratch(lz4b200_ctx* c, cudaStream_t st, size_t compact_bytes, size_t caps_bytes = 0, size_t wrap_bytes = 0)
{
    if (compact_bytes > c->compact_tmp.cap || caps_bytes > c->packed_caps.cap || wrap_bytes > c->wrap_tmp.cap) {
        CU(cudaDeviceSynchronize());
        CU(c->compact_tmp.reserve(compact_bytes)); CU(c->packed_caps.reserve(caps_bytes)); CU(c->wrap_tmp.reserve(wrap_bytes));
    }
    CU(cudaStreamWaitEvent(st, c->compact_done, 0));
    return LZ4B200_OK;
}

int launched(cudaError_t e, const char* what) { return e == cudaSuccess ? LZ4B200_OK : cuda_fail(e, what); }

// Decode group size from the ratio compressed/raw of a batch (tools/sweep.py): incompressible data is long literal runs
// (whole warps, 128-bit copies), nearly-empty streams are long matches, everything between is sequence-dense (the
// denser, the smaller the group: 8 lanes around ratio 0.58, 4 lanes around 0.37; both output-staged).
int lanes_for_ratio(double ratio, int64_t n_blocks, const DeviceInfo& dev)
{
    const int g = decode_lanes_for_ratio(ratio);
    // token-dense + at least half a wave of blocks: one lane per block (decode.cu lpb_pays; host chunks rarely fill whole
    // waves, so the middle class stays with the 8-lane group kernel)
    return g == 104 && n_blocks >= (int64_t)dev.num_sms * 32 * 8 ? 1 : g;
}

// hc_large: blocks above 64 KiB in an HC batch (-1 = not known: a device-memory batch)
int run_device(lz4b200_ctx* c, const BatchArgs& a, Op op, cudaStream_t st, int lanes = 0, int32_t hc_large = -1)
{
    if (!lanes) lanes = c->pinned_lanes();
    cudaError_t e = cudaSuccess;
    switch (op) {
    case Op::ENCODE_FAST: e = launch_encode_fast(a, c->counter(), c->encode_ctas_per_sm, c->encode_tune, c->encode_variant, c->dev, st, &c->launches); break;
    case Op::ENCODE_HC: {
        const int conc = (int)std::min<int64_t>(c->hc_concurrency, std::max(a.n_blocks, 1));
        const size_t need = c->hc_kernel < 0 ? hc_auto_scratch_bytes(a.n_blocks, hc_large, c->dev)
                          : (c->hc_kernel ? hcw_scratch_bytes(a.n_blocks, hc_large, c->hc_kernel, c->hc_warps_per_sm, c->dev) : hc_scratch_bytes(conc));
        if (need > c->hc_arena.cap) {
            CU(cudaDeviceSynchronize());           // the arena may still be in use by an earlier launch
            CU(c->hc_arena.reserve(need));
        }
        // one arena per context: an HC launch may not overlap the previous one, whatever stream it was given
        CU(cudaStreamWaitEvent(st, c->hc_done, 0));
        e = c->hc_kernel < 0 ? launch_encode_hc_auto(a, c->hc_arena.p, hc_large, c->counter(), c->dev, st, &c->launches)
          : c->hc_kernel ? launch_encode_hcw(a, c->hc_arena.p, c->hc_kernel, c->hc_warps_per_sm, hc_large, c->counter(), c->dev, st, &c->launches)
                              : launch_encode_hc(a, c->hc_arena.p, conc, c->counter(), c->dev, st, &c->launches);
        if (e == cudaSuccess) e = cudaEventRecord(c->hc_done, st);
        break;
    }
    case Op::DECODE_KNOWN:
    case Op::DECODE_UNKNOWN: e = launch_decode(a, op == Op::DECODE_KNOWN, lanes, c->counter(), c->dev, st, &c->launches); break;
    case Op::MEASURE_KNOWN:
    case Op::MEASURE_UNKNOWN: e = launch_measure(a, op == Op::MEASURE_KNOWN, c->dev, st, &c->launches); break;
    }
    return launched(e, "kernel launch");
}

// A Wrap of the batch a into whole packets: prep (each payload behind its header's place, capacity = its input length,
// LZ4Codec.cs:518-523) -> the batch codec, unchanged, on the codec's view w -> finish (the headers, the stored inputs,
// out_len = the packet sizes).
int run_wrap(lz4b200_ctx* c, const BatchArgs& a, const WrapScratch& w, Op op, cudaStream_t st, int32_t hc_large)
{
    int rc = launched(launch_wrap_prep(a, w, st, &c->launches), "wrap prep launch"); if (rc) return rc;
    const BatchArgs enc{a.src, a.src_off, w.len, a.dst, w.off, w.cap, w.res, a.n_blocks};
    rc = run_device(c, enc, op, st, 0, hc_large); if (rc) return rc;
    return launched(launch_wrap_finish(a, w, st, &c->launches), "wrap finish launch");
}

// Host-memory batch: chunks of at most host_chunk_bytes (src + dst bytes) go through the slots in turn, and a slot's
// outputs land in the caller's memory when the slot comes round again, so chunks overlap and land in block order.  On the
// device the output slots of a chunk are dense: block i starts at the sum of dst_cap over the earlier blocks of its
// chunk, so slots adjacent in dst are adjacent there too.  The measure pass has no output: its chunks are weighed by
// src_len alone, dst_cap may be null (INT32_MAX per block), and only out_len comes back (NONE).
// Only bytes a block PRODUCED ever reach the caller's buffer (the reference's safe codec leaves everything behind the
// return value untouched, its native ones spill at most 7 bytes).  A chunk's outputs land in one of four ways:
//  PER_BLOCK  chunks of at most 8 blocks: one copy per block to dst + dst_off[i];
//  RUNS       known-size decodes, which produce exactly dst_cap[i] bytes per block: one copy per maximal run of slots
//             adjacent in dst, straight into dst when it is page-locked, else through the slot's pinned buffer;
//  SCATTER    encoders and the unknown-size decoder: compacted on the device, one copy of exactly the produced bytes
//             into the slot's pinned buffer, scattered to dst + dst_off[i] from there;
//  APPEND     the packed forms (dst_off == nullptr): compacted likewise, or framed (STREAM_ENCODE), and appended at
//             dst + written (straight into dst when it is page-locked); out_off[i] receives block i's offset there,
//             out_off[n] the total.
// Mixed memory: src_dev = the source is already device memory (the kernels read the caller's buffer at the caller's
// offsets; nothing is staged), dst_dev = the destination is device memory (the kernels write the caller's slots in place;
// nothing is compacted or landed, only out_len comes back: NONE).  A chunk is weighed by what it stages, so the slots'
// device buffers stay within host_chunk_bytes whatever the batch.  The slots start behind everything enqueued on
// `caller` before the call: a producer of src, or a reader of dst's old contents.
// PLACED_DECODE (dst_dev, dst_off == nullptr, out_off set; lz4_packed.cuh): nobody stored the decoded sizes, so a stage
// measures its blocks, scans the sizes and places its blocks behind the earlier stages' -- the running total is carried
// from stage to stage in the context's `carry` cells, the slot's is the one its stage leaves -- then decodes them in place
// behind the stage's "fits" flag.  Only the placement steps are chained (the slot's `carried` event, waited on by the next
// stage's stream); everything else of neighbouring stages overlaps as in any other call.  out_off[i] receives block i's
// offset, out_off[n] the total, whether it fits dst_total_cap or not.
int run_host(lz4b200_ctx* c, Stage kind, Op op, const uint8_t* src, const int64_t* src_off, const int32_t* src_len, uint8_t* dst,
             const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, int64_t* out_off,
             int64_t dst_total_cap, bool src_dev = false, bool dst_dev = false, cudaStream_t caller = nullptr,
             const uint8_t* stored = nullptr)
{
    const bool measure = is_measure(op), framed = kind == Stage::FRAMED_DECODE, placed = kind == Stage::PLACED_DECODE;
    for (int32_t i = 0; i < n; i++)
        if (src_len[i] < 0 || (dst_cap && dst_cap[i] < 0)) return fail(LZ4B200_E_ARG, "negative block length");
    const bool src_pageable = !src_dev && is_pageable(src), dst_pageable = !measure && !dst_dev && is_pageable(dst);
    enum Mode { NONE, PER_BLOCK, RUNS, SCATTER, APPEND };
    struct Pending { int32_t b0, b1; Mode mode; };
    Pending pend[NSLOT]; bool busy[NSLOT] = {false, false, false};
    int32_t b0 = 0; int k = 0; int64_t written = 0;
    // whatever happens, nothing of this call is still in flight when it returns (the staging buffers are reused)
    struct Drain { lz4b200_ctx* c; ~Drain() { for (int i = 0; i < NSLOT; i++) cudaStreamSynchronize(c->slot[i].stream); } } drain{c};
    if (src_dev || dst_dev) {
        CU(cudaEventRecord(c->entry, caller));
        for (int i = 0; i < NSLOT; i++) CU(cudaStreamWaitEvent(c->slot[i].stream, c->entry, 0));
    }

    // RUNS: fn(offset in dst, offset in the chunk's dense layout, bytes) for every non-empty maximal run of adjacent slots
    auto for_runs = [&](int32_t c0, int32_t c1, const int64_t* dof, const std::function<int(int64_t, int64_t, size_t)>& fn) -> int {
        for (int32_t r0 = c0, i = c0 + 1; i <= c1; i++) {
            if (i < c1 && dst_off[i] == dst_off[i - 1] + dst_cap[i - 1]) continue;
            const int64_t bytes = dst_off[i - 1] + dst_cap[i - 1] - dst_off[r0];
            if (bytes > 0) { int rc = fn(dst_off[r0], dof[r0 - c0], (size_t)bytes); if (rc) return rc; }
            r0 = i;
        }
        return LZ4B200_OK;
    };

    auto retire = [&](int s) -> int {
        // the lengths (and compacted offsets) of slot s are on the host once its event has fired; land its outputs
        if (!busy[s]) return LZ4B200_OK;
        busy[s] = false;
        Slot& sl = c->slot[s];
        const Pending& p = pend[s];
        const int32_t m = p.b1 - p.b0;
        const Meta h(sl.hmeta.p, m);
        CU(cudaEventSynchronize(sl.done));
        const int64_t total = p.mode >= SCATTER ? h.off[m] : 0;
        if (p.mode == APPEND && written + total > dst_total_cap) return fail(LZ4B200_E_ARG, "packed destination too small");
        std::memcpy(out_len + p.b0, h.out, sizeof(int32_t) * (size_t)m);
        if (p.mode == PER_BLOCK) {
            for (int32_t i = 0; i < m; i++) {
                // a known-size decode produced dst_cap bytes when it succeeded, a stored copy (aux > 0: the decoder saw
                // the neutral entry and failed it) always
                const int32_t b = p.b0 + i, r = h.out[i];
                const int64_t nbytes = op == Op::DECODE_KNOWN ? (r >= 0 || (framed && h.aux[i] > 0) ? dst_cap[b] : 0) : std::max(r, 0);
                if (nbytes > 0)
                    CU(cudaMemcpyAsync(dst + dst_off[b], (uint8_t*)sl.dst.p + h.dof[i], (size_t)nbytes, cudaMemcpyDeviceToHost, sl.stream));
            }
            CU(cudaStreamSynchronize(sl.stream));
        } else if (p.mode == RUNS) {
            // the runs are in dst already, or in the slot's pinned buffer in the dense layout
            if (dst_pageable)
                return for_runs(p.b0, p.b1, h.dof, [&](int64_t to, int64_t from, size_t bytes) {
                    par_memcpy(dst + to, (const uint8_t*)sl.hout.p + from, bytes);
                    return LZ4B200_OK;
                });
        } else if (total > 0) {
            const bool direct = p.mode == APPEND && !dst_pageable;
            if (!direct) CU(sl.hout.reserve((size_t)total));
            CU(cudaMemcpyAsync(direct ? dst + written : sl.hout.p, sl.packed.p, (size_t)total, cudaMemcpyDeviceToHost, sl.stream));
            CU(cudaStreamSynchronize(sl.stream));
            const uint8_t* staged = (const uint8_t*)sl.hout.p;
            if (p.mode == SCATTER) {
                par_ranges((size_t)m, total >= (int64_t)STAGE_PARALLEL_MIN ? 1 : (size_t)m + 1, [&](size_t lo, size_t hi) {
                    for (size_t i = lo; i < hi; i++) {
                        const int64_t nb = h.off[i + 1] - h.off[i];
                        if (nb > 0) std::memcpy(dst + dst_off[p.b0 + (int32_t)i], staged + h.off[i], (size_t)nb);
                    }
                });
            } else if (!direct) {
                par_memcpy(dst + written, staged, (size_t)total);
            }
        }
        if (placed) {
            std::memcpy(out_off + p.b0, h.dof, sizeof(int64_t) * (size_t)m);
            written = h.off[0];
        }
        if (p.mode == APPEND) {
            for (int32_t i = 0; i < m; i++) out_off[p.b0 + i] = written + h.off[i];
            written += total;
        }
        return LZ4B200_OK;
    };

    while (b0 < n) {
        // ---- pick the chunk [b0, b1): bounded staged src + dst bytes ----
        int64_t bytes = 0; int32_t b1 = b0;
        while (b1 < n) {
            const int64_t w = (src_dev ? 0 : (int64_t)src_len[b1]) + (measure || dst_dev ? 0 : dst_cap[b1]);
            if (b1 > b0 && bytes + w > (int64_t)c->host_chunk_bytes) break;
            bytes += w; b1++;
        }
        const int s = k % NSLOT; k++;
        int rc = retire(s); if (rc) return rc;
        Slot& sl = c->slot[s];
        const int32_t m = b1 - b0;
        const Mode mode = measure || dst_dev ? NONE : !dst_off ? APPEND : m <= 8 ? PER_BLOCK : op == Op::DECODE_KNOWN ? RUNS : SCATTER;
        CU(sl.meta.reserve((size_t)m * (kind == Stage::WRAP_ENCODE ? WRAP_META_BYTES : META_BYTES) + (placed ? sizeof(int64_t) : 0)));
        CU(sl.hmeta.reserve((size_t)m * META_BYTES + sizeof(int64_t) * (size_t)(m + 2)));
        const Meta h(sl.hmeta.p, m), d(sl.meta.p, m);
        int64_t slo = 0, shi = 0, dsum = 0;
        if (!src_dev) {
            slo = INT64_MAX; shi = INT64_MIN;
            for (int32_t i = b0; i < b1; i++) { slo = std::min(slo, src_off[i]); shi = std::max(shi, src_off[i] + src_len[i]); }
        }
        for (int32_t i = 0; i < m; i++) {
            h.so[i] = src_off[b0 + i] - slo;
            if (dst_dev) h.dof[i] = placed ? 0 : dst_off[b0 + i];
            else { h.dof[i] = dsum; dsum += measure ? 0 : dst_cap[b0 + i]; }
            h.sl[i] = src_len[b0 + i]; h.dc[i] = dst_cap ? dst_cap[b0 + i] : INT32_MAX;
            if (framed) {
                const bool st = stored[b0 + i] != 0;
                h.aux[i] = st ? h.sl[i] : 0;
                if (st) h.sl[i] = h.dc[i] = 0;
            }
        }
        const size_t sbytes = (size_t)(shi - slo);
        if (!src_dev) CU(sl.src.reserve(sbytes + 64));
        if (!dst_dev) CU(sl.dst.reserve((size_t)dsum + 64));
        // up: the four arrays the kernels read, and a framed decode's stored lengths
        const size_t up = (size_t)((uint8_t*)(framed ? h.out : h.aux) - (uint8_t*)h.so);
        CU(cudaMemcpyAsync(sl.meta.p, sl.hmeta.p, up, cudaMemcpyHostToDevice, sl.stream));
        if (sbytes) {
            const uint8_t* from = src + slo;
            if (src_pageable && m > 8) { CU(sl.hsrc.reserve(sbytes)); par_memcpy(sl.hsrc.p, from, sbytes); from = (const uint8_t*)sl.hsrc.p; }
            CU(cudaMemcpyAsync(sl.src.p, from, sbytes, cudaMemcpyHostToDevice, sl.stream));
        }
        const BatchArgs a{src_dev ? src : (const uint8_t*)sl.src.p, d.so, d.sl, dst_dev ? dst : (uint8_t*)sl.dst.p, d.dof, d.dc, d.out, m};
        int lanes = 0;
        if (is_decode(op) && c->decode_lanes_auto && !placed) {      // (a placed stage's decoded size is known on the device only)
            double cs = 0, rs = 0;
            for (int32_t i = b0; i < b1; i++) { cs += src_len[i]; rs += dst_cap[i]; }
            lanes = lanes_for_ratio(rs > 0 ? cs / rs : 1.0, m, c->dev);
        }
        int32_t hc_large = 0;
        if (op == Op::ENCODE_HC) for (int32_t i = b0; i < b1; i++) hc_large += src_len[i] > 65536;
        switch (kind) {
        case Stage::CODEC:
        case Stage::STREAM_ENCODE:
            rc = run_device(c, a, op, sl.stream, lanes, hc_large);
            break;
        case Stage::WRAP_ENCODE:
            rc = run_wrap(c, a, wrap_scratch_at((uint8_t*)sl.meta.p + WRAP_META_OFFSET * (size_t)m, m), op, sl.stream, hc_large);
            break;
        case Stage::FRAMED_DECODE:
            rc = run_device(c, a, op, sl.stream, lanes);
            if (!rc) rc = launched(launch_stream_stored(a, d.aux, sl.stream, &c->launches), "stored copy launch");
            break;
        case Stage::PLACED_DECODE: {
            // measure -> scan -> placement, behind the previous stage's -> decode behind the stage's flag
            CU(sl.offs.reserve(sizeof(int64_t) * (size_t)(m + 1))); CU(sl.scan.reserve(compact_tmp_bytes(m)));
            const int prev = (s + NSLOT - 1) % NSLOT;
            int* fits = (int*)d.off;
            BatchArgs sizes = a; sizes.dst_cap = nullptr;
            cudaError_t e = launch_measure(sizes, false, c->dev, sl.stream, &c->launches);
            if (e == cudaSuccess) e = launch_compact(nullptr, nullptr, d.out, nullptr, (int64_t*)sl.offs.p, m, sl.scan.p, sl.scan.cap, c->dev, sl.stream, &c->launches);
            if (e != cudaSuccess) return cuda_fail(e, "packed measure launch");
            if (b0 > 0) CU(cudaStreamWaitEvent(sl.stream, c->slot[prev].carried, 0));
            e = launch_packed_prep(d.out, (const int64_t*)sl.offs.p, m, dst_total_cap, PACKED_ROOM_UNKNOWN, d.dc, fits, sl.stream, &c->launches,
                                   b0 > 0 ? c->carry + prev : nullptr, d.dof, c->carry + s);
            if (e != cudaSuccess) return cuda_fail(e, "packed placement launch");
            CU(cudaEventRecord(sl.carried, sl.stream));
            e = launch_decode(a, false, c->pinned_lanes(), c->counter(), c->dev, sl.stream, &c->launches, fits);
            if (e != cudaSuccess) return cuda_fail(e, "packed decode launch");
            CU(cudaMemcpyAsync(h.dof, d.dof, sizeof(int64_t) * (size_t)m, cudaMemcpyDeviceToHost, sl.stream));
            CU(cudaMemcpyAsync(h.off, c->carry + s, sizeof(int64_t), cudaMemcpyDeviceToHost, sl.stream));
            break;
        }
        }
        if (rc) return rc;
        if (mode >= SCATTER) {
            // the outputs back to back: compacted, or an LZ4Stream encode's frames (sizes -> scan -> headers + payloads)
            const bool frames = kind == Stage::STREAM_ENCODE;
            CU(sl.packed.reserve((size_t)dsum + (frames ? (size_t)m * STREAM_HEADER_MAX : 0) + 64));
            CU(sl.offs.reserve(sizeof(int64_t) * (size_t)(m + 1))); CU(sl.scan.reserve(compact_tmp_bytes(m)));
            uint8_t* packed = (uint8_t*)sl.packed.p;
            int64_t* offs = (int64_t*)sl.offs.p;
            cudaError_t e;
            if (frames) {
                e = launch_stream_frame_size(a, d.aux, sl.stream, &c->launches);
                if (e == cudaSuccess) e = launch_compact(nullptr, nullptr, d.aux, nullptr, offs, m, sl.scan.p, sl.scan.cap, c->dev, sl.stream, &c->launches);
                if (e == cudaSuccess) e = launch_stream_frame(a, op == Op::ENCODE_HC, packed, offs, sl.stream, &c->launches);
            } else {
                e = launch_compact(a.dst, a.dst_off, a.out_len, packed, offs, m, sl.scan.p, sl.scan.cap, c->dev, sl.stream, &c->launches);
            }
            rc = launched(e, frames ? "stream frame launch" : "compact launch"); if (rc) return rc;
            CU(cudaMemcpyAsync(h.off, offs, sizeof(int64_t) * (size_t)(m + 1), cudaMemcpyDeviceToHost, sl.stream));
        }
        CU(cudaMemcpyAsync(h.out, a.out_len, sizeof(int32_t) * (size_t)m, cudaMemcpyDeviceToHost, sl.stream));
        if (mode == RUNS) {
            if (dst_pageable) CU(sl.hout.reserve((size_t)dsum));
            rc = for_runs(b0, b1, h.dof, [&](int64_t to, int64_t from, size_t bytes) {
                CU(cudaMemcpyAsync(dst_pageable ? (uint8_t*)sl.hout.p + from : dst + to, (uint8_t*)sl.dst.p + from, bytes,
                                   cudaMemcpyDeviceToHost, sl.stream));
                return LZ4B200_OK;
            });
            if (rc) return rc;
        }
        CU(cudaEventRecord(sl.done, sl.stream));
        pend[s] = Pending{b0, b1, mode}; busy[s] = true;
        b0 = b1;
    }
    for (int i = 0; i < NSLOT; i++) { int rc = retire((k + i) % NSLOT); if (rc) return rc; }
    if (out_off) out_off[n] = written;
    return LZ4B200_OK;
}

// The side of a mixed-memory call that must be device memory is memory of the context's device (plain or managed); the
// side that must be host memory is not device memory (pageable, page-locked or managed host memory all copy).
int check_side(const lz4b200_ctx* c, const void* p, bool device, const char* what)
{
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); a.type = cudaMemoryTypeUnregistered; }
    const bool on_device = a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
    if (device && !(on_device && a.device == c->device))
        return fail(LZ4B200_E_ARG, std::string(what) + " must be device memory of the context's GPU");
    if (!device && a.type == cudaMemoryTypeDevice) return fail(LZ4B200_E_ARG, std::string(what) + " must be host memory");
    return LZ4B200_OK;
}

// Argument checks, the context's lock and its device for every batch call.  dst_off == nullptr with out_off set is the
// packed encode (lz4b200_encode_batch_packed, or its _from_device form with MEM_DEVICE_TO_HOST); the measure pass has no
// dst, dst_off or out_off.
int batch(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
          const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, Op op, int mem, void* stream,
          int64_t* out_off = nullptr, int64_t dst_total_cap = 0)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0) return fail(LZ4B200_E_ARG, "negative block count");
    if (n == 0) return LZ4B200_OK;
    const bool measure = is_measure(op);
    if (!src_off || !src_len || !out_len || !src || (!measure && (!(dst_off || out_off) || !dst_cap || !dst)))
        return fail(LZ4B200_E_ARG, "null argument");
    CallGuard g(c); if (g.rc) return g.rc;
    if (mem == LZ4B200_MEM_DEVICE) {
        BatchArgs a{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, dst_off, dst_cap, out_len, n};
        return run_device(c, a, op, (cudaStream_t)stream);
    }
    const bool src_dev = mem == LZ4B200_MEM_DEVICE_TO_HOST, dst_dev = mem == LZ4B200_MEM_HOST_TO_DEVICE;
    if (mem != LZ4B200_MEM_HOST && !src_dev && !dst_dev)
        return fail(LZ4B200_E_ARG, "mem must be LZ4B200_MEM_HOST, _DEVICE, _DEVICE_TO_HOST or _HOST_TO_DEVICE");
    if (src_dev || dst_dev) {
        // the measure pass has no destination: MEM_HOST and MEM_DEVICE already cover both places its source can be
        if (measure) return fail(LZ4B200_E_ARG, "measure_batch takes LZ4B200_MEM_HOST or LZ4B200_MEM_DEVICE");
        int rc = check_side(c, src, src_dev, "src"); if (rc) return rc;
        rc = check_side(c, dst, dst_dev, "dst"); if (rc) return rc;
    }
    return run_host(c, Stage::CODEC, op, (const uint8_t*)src, src_off, src_len, (uint8_t*)dst, dst_off, dst_cap, out_len, n, out_off,
                    dst_total_cap, src_dev, dst_dev, (cudaStream_t)stream);
}

// The single-block entry points are re-entrant like the reference's (SURVEY 8b "Threading"): every calling thread gets
// a context of its own (streams + staging buffers), created on first use and destroyed with the thread.
struct ThreadCtx {
    lz4b200_ctx* c = nullptr;
    ~ThreadCtx() { if (c) lz4b200_destroy(c); }
};
thread_local ThreadCtx g_thread_ctx;

lz4b200_ctx* default_ctx()
{
    if (!g_thread_ctx.c) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
        if (lz4b200_create(&g_thread_ctx.c, dev) != LZ4B200_OK) g_thread_ctx.c = nullptr;
    }
    return g_thread_ctx.c;
}

int single(const char* source, char* dest, int isize, int ocap, Op op)
{
    const int failed = is_encode(op) ? 0 : -1;     // encoders report failure (0), decoders an error (<0)
    lz4b200_ctx* c = default_ctx();
    if (!c || !source || !dest || isize < 0 || ocap < 0) return failed;
    int64_t so = 0, dof = 0; int32_t sl = isize, dc = ocap, out = failed;
    // zero-length buffers still need valid pointers for the staging copies
    int rc = batch(c, source, &so, &sl, dest, &dof, &dc, &out, 1, op, LZ4B200_MEM_HOST, nullptr);
    if (rc != LZ4B200_OK) return failed;
    return out;
}

// The LZ4Stream calls run the pipeline over at most this many chunks at a time: it bounds the host metadata by chunk
// count (tiny blocks would otherwise need gigabytes of it), while a call covers many pipeline stages.
constexpr int64_t STREAM_RUN_CHUNKS = 1 << 20;

// The LZ4Stream of n bytes in host or device memory (src_dev), written into host memory: each run of chunks is encoded
// (capacity = the chunk's length, LZ4Stream.cs:243-246) and its frames land back to back (STREAM_ENCODE, APPEND).  Returns
// the stream's size.  Only a chunk whose frame does not fit an int32 is refused for its size.
int64_t stream_encode(lz4b200_ctx* c, const void* src, int64_t n, int32_t block_size, int high_compression, void* dst,
                      int64_t dst_cap, bool src_dev, void* stream)
{
    if (!c || n < 0 || block_size < 1 || (n > 0 && (!src || !dst))) return fail(LZ4B200_E_ARG, "bad argument");
    if (std::min<int64_t>(block_size, n) > INT32_MAX - STREAM_HEADER_MAX) return fail(LZ4B200_E_ARG, "a chunk's frame must fit an int32");
    if (dst_cap < lz4b200_stream_bound(n, block_size)) return fail(LZ4B200_E_ARG, "dst_cap < lz4b200_stream_bound(n, block_size)");
    if (n == 0) return 0;
    CallGuard g(c); if (g.rc) return g.rc;
    if (src_dev) {
        int rc = check_side(c, src, true, "src"); if (rc) return rc;
        rc = check_side(c, dst, false, "dst"); if (rc) return rc;
    }
    const int64_t chunks = (n + block_size - 1) / block_size;
    std::vector<int64_t> so, at; std::vector<int32_t> len, res;
    int64_t w = 0;
    for (int64_t c0 = 0; c0 < chunks; c0 += STREAM_RUN_CHUNKS) {
        const int32_t m = (int32_t)std::min(STREAM_RUN_CHUNKS, chunks - c0);
        so.resize(m); len.resize(m); res.assign(m, 0); at.assign((size_t)m + 1, 0);
        for (int32_t i = 0; i < m; i++) {
            so[i] = (c0 + i) * block_size;
            len[i] = (int32_t)std::min<int64_t>(block_size, n - so[i]);
        }
        int rc = run_host(c, Stage::STREAM_ENCODE, encode_op(high_compression != 0), (const uint8_t*)src, so.data(), len.data(),
                          (uint8_t*)dst + w, nullptr, len.data(), res.data(), m, at.data(), dst_cap - w, src_dev, false,
                          (cudaStream_t)stream);
        if (rc) return rc;
        w += at[m];
    }
    return w;
}

// The LZ4Stream of n bytes in host memory, decoded into host or device memory (dst_dev).  The whole header walk comes
// before any device work, so a malformed stream writes nothing.  Returns the decoded size.
int64_t stream_decode(lz4b200_ctx* c, const void* src, int64_t n, void* dst, int64_t dst_cap, bool dst_dev, void* stream)
{
    if (!c || n < 0 || (n > 0 && !src)) return fail(LZ4B200_E_ARG, "bad argument");
    CallGuard g(c); if (g.rc) return g.rc;
    if (dst_dev) { int rc = check_side(c, src, false, "src"); if (rc) return rc; }
    std::vector<StreamChunk> chunks;
    const int64_t total = stream_walk((const uint8_t*)src, n, &chunks);
    if (total < 0) return fail((int)total, "malformed LZ4Stream");
    if (total > dst_cap || (total > 0 && !dst)) return fail(LZ4B200_E_ARG, "dst_cap < the decoded size");
    if (total == 0) return 0;
    if (dst_dev) { int rc = check_side(c, dst, true, "dst"); if (rc) return rc; }
    // one entry per non-empty chunk; the flag is the header's (a compressed chunk may have compLen == rawLen, LZ4Stream.cs:288)
    std::vector<int64_t> so, dof; std::vector<int32_t> len, raw, res; std::vector<uint8_t> stored;
    int64_t pos = 0;
    for (const StreamChunk& k : chunks) {
        if (k.raw > 0) { so.push_back(k.payload); len.push_back(k.stored); dof.push_back(pos); raw.push_back(k.raw); stored.push_back(!k.compressed); }
        pos += k.raw;
    }
    const int64_t entries = (int64_t)so.size();
    for (int64_t e0 = 0; e0 < entries; e0 += STREAM_RUN_CHUNKS) {
        const int32_t m = (int32_t)std::min(STREAM_RUN_CHUNKS, entries - e0);
        res.assign(m, -1);
        int rc = run_host(c, Stage::FRAMED_DECODE, Op::DECODE_KNOWN, (const uint8_t*)src, so.data() + e0, len.data() + e0,
                          (uint8_t*)dst, dof.data() + e0, raw.data() + e0, res.data(), m, nullptr, 0, false, dst_dev,
                          (cudaStream_t)stream, stored.data() + e0);
        if (rc) return rc;
        // a compressed chunk decodes from exactly its compLen bytes (LZ4Codec.Safe.cs:539-542)
        for (int32_t i = 0; i < m; i++)
            if (!stored[e0 + i] && res[i] != len[e0 + i]) return fail(LZ4B200_E_FORMAT, "a chunk does not decode to its compressed length");
    }
    return total;
}

// The Wrap packets of inputs in host or device memory (src_dev), landed in host memory: in the caller's slots, or packed
// (dst_off == nullptr, out_off as in the packed encode).  Every argument is checked before any device work: a negative
// length or a slot too small for its packet fails the whole call.
int wrap_packets(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, int high_compression,
                 void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n,
                 int64_t* out_off, int64_t dst_total_cap, bool src_dev, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0) return fail(LZ4B200_E_ARG, "negative packet count");
    if (n == 0) { if (out_off) out_off[0] = 0; return LZ4B200_OK; }
    if (!src || !src_off || !src_len || !dst || !out_len || (dst_off ? !dst_cap : !out_off)) return fail(LZ4B200_E_ARG, "null argument");
    // the slots' dense layout holds packets, whatever room the caller's slots have
    std::vector<int32_t> pcap((size_t)n);
    for (int32_t i = 0; i < n; i++) {
        if (src_len[i] < 0 || src_len[i] > INT32_MAX - WRAP_HEADER) return fail(LZ4B200_E_ARG, "input length: negative, or a packet above INT32_MAX bytes");
        if (dst_off && (int64_t)dst_cap[i] < (int64_t)src_len[i] + WRAP_HEADER) return fail(LZ4B200_E_ARG, "dst_cap[i] < src_len[i] + 8");
        pcap[i] = src_len[i] + WRAP_HEADER;
    }
    CallGuard g(c); if (g.rc) return g.rc;
    if (src_dev) {
        int rc = check_side(c, src, true, "src"); if (rc) return rc;
        rc = check_side(c, dst, false, "dst"); if (rc) return rc;
    }
    return run_host(c, Stage::WRAP_ENCODE, encode_op(high_compression != 0), (const uint8_t*)src, src_off, src_len, (uint8_t*)dst,
                    dst_off, pcap.data(), out_len, n, out_off, dst_total_cap, src_dev, false, (cudaStream_t)stream);
}

// Unwrap n packets in host memory into host or device memory (dst_dev): into the caller's slots, or packed (dst_off ==
// nullptr: packet i at out_off[i], the prefix sum of the sizes, out_off[n] the total; nothing is restored and out_len holds
// the sizes when the total exceeds dst_total_cap).  The headers are read first, by several threads: small packets far
// apart in a large batch cost a cache and TLB miss each, and one thread would then take longer than the link.  A rejected
// packet gets its status before any device work (E_FORMAT, or E_ARG above its capacity), an empty one 0.  Every other
// packet is one entry of a known-size decode: a compressed one decodes its stored bytes into raw bytes, a stored one is
// copied (FRAMED_DECODE).
int unwrap_packets(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                   const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, int64_t* out_off,
                   int64_t dst_total_cap, bool dst_dev, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0) return fail(LZ4B200_E_ARG, "negative packet count");
    if (n == 0) { if (out_off) out_off[0] = 0; return LZ4B200_OK; }
    if (!src || !src_off || !src_len || !dst || !out_len || (dst_off ? !dst_cap : !out_off)) return fail(LZ4B200_E_ARG, "null argument");
    CallGuard g(c); if (g.rc) return g.rc;
    if (dst_dev) {
        int rc = check_side(c, src, false, "src"); if (rc) return rc;
        rc = check_side(c, dst, true, "dst"); if (rc) return rc;
    }
    const uint8_t* s = (const uint8_t*)src;
    struct Header { int32_t raw, stored, size; };
    std::vector<Header> hdr((size_t)n);
    par_ranges((size_t)n, 4096, [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; i++) hdr[i].size = read_header(s + src_off[i], src_len[i], &hdr[i].raw, &hdr[i].stored);
    });
    std::vector<int32_t> sizes;
    if (!dst_off) {
        sizes.resize((size_t)n);
        int64_t total = 0;
        for (int32_t i = 0; i < n; i++) {
            out_len[i] = hdr[i].size;
            sizes[i] = std::max(hdr[i].size, 0);
            out_off[i] = total;
            total += sizes[i];
        }
        out_off[n] = total;
        if (total > dst_total_cap) return LZ4B200_OK;
        dst_off = out_off; dst_cap = sizes.data();
    }
    std::vector<int64_t> so, dof; std::vector<int32_t> len, cap, res, idx; std::vector<uint8_t> stored;
    for (int32_t i = 0; i < n; i++) {
        const Header& h = hdr[i];
        out_len[i] = h.size >= 0 && h.size > dst_cap[i] ? LZ4B200_E_ARG : h.size;
        if (out_len[i] <= 0) continue;
        so.push_back(src_off[i] + WRAP_HEADER); len.push_back(h.stored); dof.push_back(dst_off[i]); cap.push_back(h.size);
        stored.push_back(h.stored >= h.raw); idx.push_back(i);
    }
    if (so.empty()) return LZ4B200_OK;
    const int32_t m = (int32_t)so.size();
    res.assign((size_t)m, -1);
    int rc = run_host(c, Stage::FRAMED_DECODE, Op::DECODE_KNOWN, s, so.data(), len.data(), (uint8_t*)dst, dof.data(), cap.data(),
                      res.data(), m, nullptr, 0, false, dst_dev, (cudaStream_t)stream, stored.data());
    if (rc) return rc;
    // a compressed packet decodes from exactly its stored bytes (LZ4Codec.cs:595); one that does not is that packet's
    // E_FORMAT, not the call's
    for (int32_t j = 0; j < m; j++)
        if (!stored[j]) out_len[idx[j]] = res[j] == len[j] ? cap[j] : LZ4B200_E_FORMAT;
    return LZ4B200_OK;
}

}  // namespace

extern "C" {

int lz4b200_version(void) { return LZ4B200_VERSION; }
const char* lz4b200_last_error(void) { return g_err.c_str(); }

int lz4b200_device_count(void)
{
    int n = 0, ok = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    for (int i = 0; i < n; i++) {
        int major = 0;
        if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, i) == cudaSuccess && major == 9) ok++;
    }
    return ok;
}

int lz4b200_compress_bound(int n) { return n < 0 ? 0 : n + n / 255 + 16; }

int lz4b200_create(lz4b200_ctx** out, int device)
{
    if (!out) return fail(LZ4B200_E_ARG, "null out pointer");
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return fail(LZ4B200_E_NODEVICE, "no CUDA device"); }
    if (device < 0 || device >= n) return fail(LZ4B200_E_ARG, "device index out of range");
    int major = 0;
    CU(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
    if (major != 9) return fail(LZ4B200_E_NODEVICE, "device is not compute capability 9.x (this library holds sm_90a code only)");
    DeviceGuard g(device);
    if (!g.ok) return fail(LZ4B200_E_CUDA, "cudaSetDevice failed");
    lz4b200_ctx* c = new lz4b200_ctx();
    c->device = device;
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device); c->dev.num_sms = v;
    cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerMultiprocessor, device); c->dev.smem_per_sm = v;
    cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, device); c->dev.smem_optin = v;
    cudaError_t e = cudaMalloc(&c->counters, sizeof(uint32_t) * NCOUNTER);
    if (e == cudaSuccess) e = cudaMalloc(&c->carry, sizeof(int64_t) * NSLOT);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->hc_done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->compact_done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->entry, cudaEventDisableTiming);
    for (int i = 0; i < NSLOT && e == cudaSuccess; i++) {
        e = cudaStreamCreateWithFlags(&c->slot[i].stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->slot[i].done, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->slot[i].carried, cudaEventDisableTiming);
    }
    if (e != cudaSuccess) { int rc = cuda_fail(e, "context creation"); lz4b200_destroy(c); return rc; }
    *out = c;
    return LZ4B200_OK;
}

void lz4b200_destroy(lz4b200_ctx* c)
{
    if (!c) return;
    DeviceGuard g(c->device);
    cudaDeviceSynchronize();
    for (Slot& s : c->slot) {
        if (s.done) cudaEventDestroy(s.done);
        if (s.carried) cudaEventDestroy(s.carried);
        if (s.stream) cudaStreamDestroy(s.stream);
    }
    if (c->hc_done) cudaEventDestroy(c->hc_done);
    if (c->compact_done) cudaEventDestroy(c->compact_done);
    if (c->entry) cudaEventDestroy(c->entry);
    if (c->counters) cudaFree(c->counters);
    if (c->carry) cudaFree(c->carry);
    delete c;                                      // (the buffers free themselves, on the context's device)
}

int lz4b200_synchronize(lz4b200_ctx* c)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    DeviceGuard g(c->device);
    for (int i = 0; i < NSLOT; i++) CU(cudaStreamSynchronize(c->slot[i].stream));
    return LZ4B200_OK;
}

int lz4b200_encode_batch(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                         const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, int mode, int mem, void* stream)
{
    if (mode != LZ4B200_MODE_FAST && mode != LZ4B200_MODE_HC) return fail(LZ4B200_E_ARG, "unknown encoder mode");
    return batch(c, src, src_off, src_len, dst, dst_off, dst_cap, out_len, n, encode_op(mode == LZ4B200_MODE_HC), mem, stream);
}

int lz4b200_encode_batch_packed(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                const int32_t* dst_cap, void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len,
                                int32_t n, int mode)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (mode != LZ4B200_MODE_FAST && mode != LZ4B200_MODE_HC) return fail(LZ4B200_E_ARG, "unknown encoder mode");
    if (n < 0 || !out_off) return fail(LZ4B200_E_ARG, "bad argument");
    if (n == 0) { out_off[0] = 0; return LZ4B200_OK; }
    return batch(c, src, src_off, src_len, dst, nullptr, dst_cap, out_len, n, encode_op(mode == LZ4B200_MODE_HC), LZ4B200_MEM_HOST,
                 nullptr, out_off, dst_total_cap);
}

int lz4b200_encode_batch_packed_from_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                            const int32_t* dst_cap, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                            int32_t* out_len, int32_t n, int mode, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (mode != LZ4B200_MODE_FAST && mode != LZ4B200_MODE_HC) return fail(LZ4B200_E_ARG, "unknown encoder mode");
    if (n < 0 || !out_off) return fail(LZ4B200_E_ARG, "bad argument");
    if (n == 0) { out_off[0] = 0; return LZ4B200_OK; }
    return batch(c, src, src_off, src_len, dst, nullptr, dst_cap, out_len, n, encode_op(mode == LZ4B200_MODE_HC),
                 LZ4B200_MEM_DEVICE_TO_HOST, stream, out_off, dst_total_cap);
}

// ---- LZ4Stream (lz4_stream.cuh): the host pipeline, the frames written on the device ----------------------------------
int64_t lz4b200_stream_encode(lz4b200_ctx* c, const void* src, int64_t n, int32_t block_size, int high_compression, void* dst,
                              int64_t dst_cap)
{
    return stream_encode(c, src, n, block_size, high_compression, dst, dst_cap, false, nullptr);
}

int64_t lz4b200_stream_decode(lz4b200_ctx* c, const void* src, int64_t n, void* dst, int64_t dst_cap)
{
    return stream_decode(c, src, n, dst, dst_cap, false, nullptr);
}

int64_t lz4b200_stream_encode_from_device(lz4b200_ctx* c, const void* src, int64_t n, int32_t block_size, int high_compression,
                                          void* dst, int64_t dst_cap, void* stream)
{
    if (block_size > INT32_MAX - STREAM_HEADER_MAX) return fail(LZ4B200_E_ARG, "block_size: a chunk's frame must fit an int32");
    return stream_encode(c, src, n, block_size, high_compression, dst, dst_cap, true, stream);
}

int64_t lz4b200_stream_decode_to_device(lz4b200_ctx* c, const void* src, int64_t n, void* dst, int64_t dst_cap, void* stream)
{
    if (c && n == 0) return 0;
    return stream_decode(c, src, n, dst, dst_cap, true, stream);
}

int lz4b200_decode_batch(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                         const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, int known_len, int mem, void* stream)
{
    return batch(c, src, src_off, src_len, dst, dst_off, dst_cap, out_len, n, known_len ? Op::DECODE_KNOWN : Op::DECODE_UNKNOWN,
                 mem, stream);
}

int lz4b200_measure_batch(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, const int32_t* dst_cap,
                          int32_t* out_len, int32_t n, int known_len, int mem, void* stream)
{
    if (known_len && !dst_cap) return fail(LZ4B200_E_ARG, "dst_cap may be NULL only when known_len == 0");
    return batch(c, src, src_off, src_len, nullptr, nullptr, dst_cap, out_len, n, known_len ? Op::MEASURE_KNOWN : Op::MEASURE_UNKNOWN,
                 mem, stream);
}

// measure -> scan -> capacities + "fits" -> decode, all enqueued on `stream`: the decoders leave at once (pick gate)
// when the total does not fit, so out_len keeps the measured sizes and dst is untouched.
int lz4b200_decode_batch_packed(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0 || !out_off || dst_total_cap < 0) return fail(LZ4B200_E_ARG, "bad argument");
    CallGuard g(c); if (g.rc) return g.rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) { CU(cudaMemsetAsync(out_off, 0, sizeof(int64_t), st)); return LZ4B200_OK; }     // out_off[0] = total = 0
    if (!src || !src_off || !src_len || !dst || !out_len) return fail(LZ4B200_E_ARG, "null argument");
    int rc = call_scratch(c, st, compact_tmp_bytes(n), sizeof(int32_t) * ((size_t)n + 1)); if (rc) return rc;
    int32_t* caps = (int32_t*)c->packed_caps.p;
    int* fits = (int*)(caps + n);
    const BatchArgs m{(const uint8_t*)src, src_off, src_len, nullptr, nullptr, nullptr, out_len, n};
    cudaError_t e = launch_measure(m, false, c->dev, st, &c->launches);
    if (e == cudaSuccess) e = launch_compact(nullptr, nullptr, out_len, nullptr, out_off, n, c->compact_tmp.p, c->compact_tmp.cap, c->dev, st, &c->launches);
    if (e == cudaSuccess) e = launch_packed_prep(out_len, out_off, n, dst_total_cap, PACKED_ROOM_UNKNOWN, caps, fits, st, &c->launches);
    if (e == cudaSuccess) {
        const BatchArgs d{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, out_off, caps, out_len, n};
        e = launch_decode(d, false, c->pinned_lanes(), c->counter(), c->dev, st, &c->launches, fits);
    }
    if (e != cudaSuccess) return cuda_fail(e, "packed decode launch");
    CU(cudaEventRecord(c->compact_done, st));
    return LZ4B200_OK;
}

// The same from host memory, through the pipeline (run_host): the sizes stay on the device, a stage at a time.
int lz4b200_decode_batch_packed_to_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                          void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n,
                                          void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0 || !out_off || dst_total_cap < 0) return fail(LZ4B200_E_ARG, "bad argument");
    if (n == 0) { out_off[0] = 0; return LZ4B200_OK; }
    if (!src || !src_off || !src_len || !dst || !out_len) return fail(LZ4B200_E_ARG, "null argument");
    CallGuard g(c); if (g.rc) return g.rc;
    int rc = check_side(c, src, false, "src"); if (rc) return rc;
    rc = check_side(c, dst, true, "dst"); if (rc) return rc;
    return run_host(c, Stage::PLACED_DECODE, Op::DECODE_UNKNOWN, (const uint8_t*)src, src_off, src_len, (uint8_t*)dst, nullptr,
                    nullptr, out_len, n, out_off, dst_total_cap, false, true, (cudaStream_t)stream);
}

int lz4b200_compact(lz4b200_ctx* c, const void* slots, const int64_t* slot_off, const int32_t* len, void* packed,
                    int64_t* out_off, int32_t n, void* stream)
{
    if (!c || !slot_off || !len || !out_off || n < 0) return fail(LZ4B200_E_ARG, "bad argument");
    CallGuard g(c); if (g.rc) return g.rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) { CU(cudaMemsetAsync(out_off, 0, sizeof(int64_t), st)); return LZ4B200_OK; }     // out_off[0] = total = 0
    int rc = call_scratch(c, st, compact_tmp_bytes(n)); if (rc) return rc;
    cudaError_t e = launch_compact((const uint8_t*)slots, slot_off, len, (uint8_t*)packed, out_off, n,
                                   c->compact_tmp.p, c->compact_tmp.cap, c->dev, st, &c->launches);
    if (e != cudaSuccess) return cuda_fail(e, "compact launch");
    CU(cudaEventRecord(c->compact_done, st));
    return LZ4B200_OK;
}

// ---- Wrap / Unwrap packets in device memory (lz4_wrap.cuh): prep -> the batch codec, unchanged -> finish, on `stream` ----
int lz4b200_wrap_batch_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, int high_compression,
                              void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0) return fail(LZ4B200_E_ARG, "negative packet count");
    CallGuard g(c); if (g.rc) return g.rc;
    if (n == 0) return LZ4B200_OK;
    if (!src || !src_off || !src_len || !dst || !dst_off || !dst_cap || !out_len) return fail(LZ4B200_E_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = call_scratch(c, st, 0, 0, n * WRAP_SCRATCH_BYTES); if (rc) return rc;
    // the same encode as lz4b200_encode_batch(MEM_DEVICE): HC sizes its arena as if every block were above 64 KiB
    const BatchArgs a{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, dst_off, dst_cap, out_len, n};
    rc = run_wrap(c, a, wrap_scratch_at(c->wrap_tmp.p, n), encode_op(high_compression != 0), st, -1); if (rc) return rc;
    CU(cudaEventRecord(c->compact_done, st));
    return LZ4B200_OK;
}

int lz4b200_unwrap_batch_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0) return fail(LZ4B200_E_ARG, "negative packet count");
    CallGuard g(c); if (g.rc) return g.rc;
    if (n == 0) return LZ4B200_OK;
    if (!src || !src_off || !src_len || !dst || !dst_off || !dst_cap || !out_len) return fail(LZ4B200_E_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    int rc = call_scratch(c, st, 0, 0, n * WRAP_SCRATCH_BYTES); if (rc) return rc;
    const WrapScratch w = wrap_scratch_at(c->wrap_tmp.p, n);
    const BatchArgs a{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, dst_off, dst_cap, out_len, n};
    cudaError_t e = launch_unwrap_prep(a, w, st, &c->launches);
    if (e != cudaSuccess) return cuda_fail(e, "unwrap prep launch");
    // the compressed packets, known size (LZ4Codec.cs:595); stored and rejected ones are neutral entries
    const BatchArgs dec{(const uint8_t*)src, w.off, w.len, (uint8_t*)dst, dst_off, w.cap, w.res, n};
    rc = run_device(c, dec, Op::DECODE_KNOWN, st); if (rc) return rc;
    e = launch_unwrap_finish(a, w, nullptr, st, &c->launches);
    if (e != cudaSuccess) return cuda_fail(e, "unwrap finish launch");
    CU(cudaEventRecord(c->compact_done, st));
    return LZ4B200_OK;
}

// sizes from the headers -> scan into out_off -> capacities + "fits" -> decode and stored copies, both behind the flag
int lz4b200_unwrap_batch_packed(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0) return fail(LZ4B200_E_ARG, "negative packet count");
    CallGuard g(c); if (g.rc) return g.rc;
    if (!out_off || dst_total_cap < 0) return fail(LZ4B200_E_ARG, "bad argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) { CU(cudaMemsetAsync(out_off, 0, sizeof(int64_t), st)); return LZ4B200_OK; }     // out_off[0] = total = 0
    if (!src || !src_off || !src_len || !dst || !out_len) return fail(LZ4B200_E_ARG, "null argument");
    int rc = call_scratch(c, st, compact_tmp_bytes(n), sizeof(int32_t) * ((size_t)n + 1), n * WRAP_SCRATCH_BYTES); if (rc) return rc;
    const WrapScratch w = wrap_scratch_at(c->wrap_tmp.p, n);
    int32_t* caps = (int32_t*)c->packed_caps.p;
    int* fits = (int*)(caps + n);
    const BatchArgs a{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, out_off, nullptr, out_len, n};
    cudaError_t e = launch_unwrap_prep(a, w, st, &c->launches);
    if (e == cudaSuccess) e = launch_compact(nullptr, nullptr, out_len, nullptr, out_off, n, c->compact_tmp.p, c->compact_tmp.cap, c->dev, st, &c->launches);
    if (e == cudaSuccess) e = launch_packed_prep(out_len, out_off, n, dst_total_cap, 0, caps, fits, st, &c->launches);
    if (e == cudaSuccess) {
        const BatchArgs dec{(const uint8_t*)src, w.off, w.len, (uint8_t*)dst, out_off, caps, w.res, n};
        e = launch_decode(dec, true, c->pinned_lanes(), c->counter(), c->dev, st, &c->launches, fits);
    }
    if (e == cudaSuccess) e = launch_unwrap_finish(a, w, fits, st, &c->launches);
    if (e != cudaSuccess) return cuda_fail(e, "packed unwrap launch");
    CU(cudaEventRecord(c->compact_done, st));
    return LZ4B200_OK;
}

// ---- Wrap / Unwrap packets with a side in host memory: the host pipeline (run_host, WRAP_ENCODE / FRAMED_DECODE) ----
int lz4b200_wrap_batch(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, int high_compression,
                       void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n)
{
    return wrap_packets(c, src, src_off, src_len, high_compression, dst, dst_off, dst_cap, out_len, n, nullptr, 0, false, nullptr);
}

int lz4b200_unwrap_batch(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                         const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n)
{
    return unwrap_packets(c, src, src_off, src_len, dst, dst_off, dst_cap, out_len, n, nullptr, 0, false, nullptr);
}

int lz4b200_wrap_batch_from_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                   int high_compression, void* dst, const int64_t* dst_off, const int32_t* dst_cap,
                                   int32_t* out_len, int32_t n, void* stream)
{
    return wrap_packets(c, src, src_off, src_len, high_compression, dst, dst_off, dst_cap, out_len, n, nullptr, 0, true, stream);
}

int lz4b200_wrap_batch_packed_from_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                          int high_compression, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                          int32_t* out_len, int32_t n, void* stream)
{
    if (!out_off) return fail(LZ4B200_E_ARG, "bad argument");
    return wrap_packets(c, src, src_off, src_len, high_compression, dst, nullptr, nullptr, out_len, n, out_off, dst_total_cap,
                        true, stream);
}

int lz4b200_unwrap_batch_to_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                   const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream)
{
    return unwrap_packets(c, src, src_off, src_len, dst, dst_off, dst_cap, out_len, n, nullptr, 0, true, stream);
}

int lz4b200_unwrap_batch_packed_to_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                          void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n,
                                          void* stream)
{
    if (!out_off || dst_total_cap < 0) return fail(LZ4B200_E_ARG, "bad argument");
    return unwrap_packets(c, src, src_off, src_len, dst, nullptr, nullptr, out_len, n, out_off, dst_total_cap, true, stream);
}

int lz4b200_synth_fill(lz4b200_ctx* c, void* dst, int64_t n_blocks, int32_t block_size, int cls, uint64_t seed,
                       int64_t first_block, void* stream)
{
    if (!c || !dst) return fail(LZ4B200_E_ARG, "bad argument");
    CallGuard g(c); if (g.rc) return g.rc;
    cudaError_t e = launch_synth((uint8_t*)dst, n_blocks, block_size, cls, seed, first_block, c->dev,
                                 (cudaStream_t)stream, &c->launches);
    if (e != cudaSuccess) return cuda_fail(e, "synth launch");
    return LZ4B200_OK;
}

int lz4b200_set_option(lz4b200_ctx* c, const char* key, int64_t value)
{
    if (!c || !key) return fail(LZ4B200_E_ARG, "bad argument");
    std::lock_guard<std::mutex> lock(c->mu);
    std::string k(key);
    if (k == "decode_lanes") {
        const int64_t g = value % 100;                 // 100 + G = the output-staged variant of the G-lane decoder
        const bool lpb = value == 1;                   // one lane per block (lz4_decode_lpb.cuh)
        if (!lpb && ((g != 4 && g != 8 && g != 16 && g != 32) || (value != g && value != 100 + g))) return fail(LZ4B200_E_ARG, "decode_lanes must be 1, 4, 8, 16, 32 (or 100 + one of the last four)");
        c->decode_lanes = (int)value; c->decode_lanes_auto = false;
    }
    else if (k == "decode_lanes_auto") { c->decode_lanes_auto = value != 0; }
    else if (k == "encode_variant") { if (value != 1 && value != 2) return fail(LZ4B200_E_ARG, "encode_variant must be 1 or 2"); c->encode_variant = (int)value; }
    else if (k == "encode_prefetch") { if (value < -65536 || value > 65536) return fail(LZ4B200_E_ARG, "encode_prefetch out of range"); c->encode_tune[0] = (int)value; }
    else if (k == "encode_lane_copy_max" || k == "encode_probe_max" || k == "encode_wide_min") {
        if (value < 0 || value > 65536) return fail(LZ4B200_E_ARG, "encoder heuristic out of range");
        c->encode_tune[k == "encode_lane_copy_max" ? 1 : (k == "encode_probe_max" ? 2 : 3)] = (int)value;
    }
    else if (k == "encode_ctas_per_sm") { if (value < 0 || value > 32) return fail(LZ4B200_E_ARG, "encode_ctas_per_sm out of range"); c->encode_ctas_per_sm = (int)value; }
    else if (k == "hc_concurrency") {
        if (value < 32 || value > (1 << 20)) return fail(LZ4B200_E_ARG, "hc_concurrency out of range");
        DeviceGuard g(c->device);
        cudaDeviceSynchronize();
        c->hc_arena.release();
        c->hc_concurrency = (int)value;
    }
    else if (k == "hc_kernel") { if (value < -1 || value > 2) return fail(LZ4B200_E_ARG, "hc_kernel must be -1 (chosen per batch), 0 (thread per block), 1 or 2 (warp per block: blocks <= 64 KiB in shared memory / read through L1)"); c->hc_kernel = (int)value; }
    else if (k == "hc_warps_per_sm") { if (value < 0 || value > 32) return fail(LZ4B200_E_ARG, "hc_warps_per_sm must be 0..32"); c->hc_warps_per_sm = (int)value; }
    else if (k == "host_chunk_mb") { if (value < 1 || value > 4096) return fail(LZ4B200_E_ARG, "host_chunk_mb out of range"); c->host_chunk_bytes = (size_t)value << 20; }
    else return fail(LZ4B200_E_ARG, "unknown option");
    return LZ4B200_OK;
}

int lz4b200_get_option(lz4b200_ctx* c, const char* key, int64_t* value)
{
    if (!c || !key || !value) return fail(LZ4B200_E_ARG, "bad argument");
    std::lock_guard<std::mutex> lock(c->mu);
    const std::string k(key);
    if (k == "hc_kernel") *value = c->hc_kernel;
    else if (k == "hc_warps_per_sm") *value = c->hc_warps_per_sm;
    else if (k == "hc_concurrency") *value = c->hc_concurrency;
    else if (k == "decode_lanes") *value = c->decode_lanes_auto ? 0 : c->decode_lanes;
    else if (k == "encode_variant") *value = c->encode_variant;
    else if (k == "encode_ctas_per_sm") *value = c->encode_ctas_per_sm;
    else return fail(LZ4B200_E_ARG, "unknown option");
    return LZ4B200_OK;
}

int64_t lz4b200_launch_count(lz4b200_ctx* c) { return c ? c->launches : 0; }

int lz4b200_host_register(void* ptr, int64_t bytes)
{
    if (!ptr || bytes <= 0) return fail(LZ4B200_E_ARG, "bad argument");
    CU(cudaHostRegister(ptr, (size_t)bytes, cudaHostRegisterPortable));
    return LZ4B200_OK;
}
int lz4b200_host_unregister(void* ptr)
{
    if (!ptr) return fail(LZ4B200_E_ARG, "bad argument");
    CU(cudaHostUnregister(ptr));
    return LZ4B200_OK;
}

int lz4b200_peer_copy(void* dst, const void* src, int64_t bytes, void* stream)
{
    if (bytes < 0 || (bytes && (!dst || !src))) return fail(LZ4B200_E_ARG, "bad argument");
    if (!bytes) return LZ4B200_OK;
    int cur = 0, dev[2];
    CU(cudaGetDevice(&cur));
    const void* ends[2] = {dst, src};
    for (int k = 0; k < 2; k++) {
        cudaPointerAttributes at{};
        CU(cudaPointerGetAttributes(&at, ends[k]));
        if (at.type != cudaMemoryTypeDevice) return fail(LZ4B200_E_ARG, "lz4b200_peer_copy: both buffers must be device memory");
        dev[k] = at.device;
    }
    for (int k = 0; k < 2; k++) {                                // both directions of the pair, once
        CU(cudaSetDevice(dev[k]));
        cudaError_t e = cudaDeviceEnablePeerAccess(dev[1 - k], 0);
        (void)cudaGetLastError();
        if (dev[0] != dev[1] && e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { cudaSetDevice(cur); return cuda_fail(e, "cudaDeviceEnablePeerAccess"); }
    }
    CU(cudaSetDevice(cur));
    CU(cudaMemcpyPeerAsync(dst, dev[0], src, dev[1], (size_t)bytes, (cudaStream_t)stream));   // a copy-engine transfer
    return LZ4B200_OK;
}

int lz4b200_compress_limitedOutput(const char* s, char* d, int isize, int cap) { return single(s, d, isize, cap, Op::ENCODE_FAST); }
int lz4b200_compressHC_limitedOutput(const char* s, char* d, int isize, int cap) { return single(s, d, isize, cap, Op::ENCODE_HC); }
int lz4b200_uncompress(const char* s, char* d, int isize, int osize) { return single(s, d, isize, osize, Op::DECODE_KNOWN); }
int lz4b200_uncompress_unknownOutputSize(const char* s, char* d, int isize, int cap) { return single(s, d, isize, cap, Op::DECODE_UNKNOWN); }

}  // extern "C"
