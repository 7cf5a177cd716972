// capi.cu -- the C ABI of liblz4b200.so (include/lz4b200.h): context, batched entry points, single-block entry points.
//
// Every call on host memory (the batches with LZ4B200_MEM_HOST, the packed encode, the measure pass, the single-block entry
// points, and the LZ4Stream and Wrap / Unwrap calls) goes through one software pipeline, run_host: the block list is cut
// into chunks, and for each chunk H2D(inputs) -> kernel -> D2H(outputs) is enqueued on one of NSLOT streams, so that the
// copy engines (both PCIe directions) and the SMs work on different chunks at the same time.  The mixed-memory batches
// (MEM_DEVICE_TO_HOST, MEM_HOST_TO_DEVICE and the packed encode from device memory) and the LZ4Stream and Wrap / Unwrap
// calls between device and host memory go through it too, skipping the copy of whichever side is already on the device;
// so does the packed unknown-size decode from host into device memory, whose output offset is carried across the stages
// on the device (Placement, lz4_packed.cuh).  What a stage runs is named by its caller (Stage) and mapped to its sequence
// in one place (run_stage); the codec operation is named by Op.
// The asynchronous calls between device memory and page-locked host memory (the packed encode, Wrap and LZ4Stream encode
// into it, the decode, packed decode, Unwrap and LZ4Stream decode from it, and the decode, Unwrap and LZ4Stream decode
// from offsets or a size the device wrote) are each one AsyncCall, which names where its stages' blocks come from
// (Source); after its own argument checks each enters through enter_async, and run_async cuts its stages by the same plan
// (or arithmetically, by chunks), runs the same stage sequences on streams and buffers of their own and returns without
// waiting.  A stage is arrival (by source), its kind's sequence (run_stage) and departure (by kind): the packed encodes'
// stages land in host memory from a kernel (lz4_land.cuh), since where a stage lands is known only on the device, the
// Unwraps read their headers on the device (run_unwrap), and the LZ4Stream encode computes its chunk tables on the device.
// The device-memory calls enter through one path (DeviceCall): each states what it takes from the context (Need), which
// admits it to a CUDA graph capture or grows an eager call's scratch; lz4b200_reserve grows to the same needs.
// The LZ4Stream frames and the Wrap headers are written on the device (lz4_stream.cuh, lz4_wrap.cuh) whichever side the
// caller's bytes are on; the host only reads headers (framing.cpp).  There is no CPU codec in this library: if the device
// or the kernel image is unusable every entry point reports an error.
#include "../../include/lz4b200.h"
#include "framing.h"
#include "kernels.h"
#include "lz4_lift.cuh"
#include "lz4_packed.cuh"
#include "lz4_stream.cuh"
#include "lz4_wrap.cuh"

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <functional>
#include <memory>
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
constexpr int NCOUNTER = 256;                 // the eager calls' ring of counter sets (four words each)
constexpr int NCAPTURED = 4096;                // counter sets for captured calls, never recycled (64 KiB behind the ring)
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

// Device scratch that a captured call may reference (the context's call scratch and HC arena).  A graph keeps the address
// it captured, so once a captured call has referenced the buffer (held), growing it retires the old buffer to the
// context's list, which lz4b200_destroy frees, instead of freeing it.  A buffer no capture referenced grows as a DevBuf.
struct SharedBuf : DevBuf {
    bool held = false;
    cudaError_t grow(size_t n, std::vector<void*>& retired)
    {
        if (n <= cap) return cudaSuccess;
        drop(retired);
        return reserve(n);
    }
    void drop(std::vector<void*>& retired)
    {
        if (held && p) { retired.push_back(p); p = nullptr; cap = 0; }
        held = false;
        release();
    }
};

// Whether a call's stream is capturing (a CUDA graph being recorded), and which capture.
struct Capture { bool on = false; unsigned long long id = 0; };

// The order of the calls that share one piece of the context's scratch, whatever streams they are on: each waits on
// `done`, then records it.  Inside a capture the wait and the record are external event nodes, so that a replay waits for
// the call enqueued before it and the call enqueued after it waits for the replay, as eager calls do.  An external wait
// sees the event as it was when the graph was launched, so captured calls of the one capture are also chained through
// `inner`, an ordinary captured record / wait, in case the capture forks them onto separate streams.  `inner` remembers
// one capture: while two threads capture calls of one context, a capture's forked calls may miss that inner order (one
// context per caller thread, include/lz4b200.h).
struct Chain {
    cudaEvent_t done = nullptr, inner = nullptr;
    unsigned long long inner_id = 0;       // the capture that last recorded `inner` (0: none)
    cudaError_t wait(cudaStream_t st, const Capture& cap) const
    {
        if (!cap.on) return cudaStreamWaitEvent(st, done, 0);
        cudaError_t e = cudaStreamWaitEvent(st, done, cudaEventWaitExternal);
        if (e == cudaSuccess && inner_id == cap.id) e = cudaStreamWaitEvent(st, inner, 0);
        return e;
    }
    cudaError_t record(cudaStream_t st, const Capture& cap)
    {
        if (!cap.on) return cudaEventRecord(done, st);
        cudaError_t e = cudaEventRecordWithFlags(done, st, cudaEventRecordExternal);
        if (e == cudaSuccess) e = cudaEventRecord(inner, st);
        if (e == cudaSuccess) inner_id = cap.id;
        return e;
    }
};

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
// What CUDA says p is: its kind of memory (cudaMemoryTypeUnregistered for pageable memory, or when CUDA cannot tell), its
// device and its device address.
cudaPointerAttributes pointer_attributes(const void* p)
{
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); a.type = cudaMemoryTypeUnregistered; }
    return a;
}
bool is_pageable(const void* p) { return pointer_attributes(p).type == cudaMemoryTypeUnregistered; }

// A stream of the pipeline and the buffers of the stage on it.  `done`: the slot's last work of the call is enqueued;
// `carried`: the stage's placement or landing step, which leaves the running total in the slot's carry cell, is enqueued
// (the packed forms); meta, offs, scan: the stage's device metadata, scan offsets and scan scratch.
struct SlotBase {
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr, carried = nullptr;
    DevBuf meta, offs, scan;
};
cudaError_t create_slot(SlotBase& s)
{
    cudaError_t e = cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s.carried, cudaEventDisableTiming);
    return e;
}
void destroy_slot(SlotBase& s)
{
    if (s.done) cudaEventDestroy(s.done);
    if (s.carried) cudaEventDestroy(s.carried);
    if (s.stream) cudaStreamDestroy(s.stream);
}

struct Slot : SlotBase {
    DevBuf src, dst, packed;
    PinBuf hmeta, hsrc, hout;              // pinned: chunk metadata, staged pageable sources, staged outputs
};

// The stages of the asynchronous calls (run_async) go through buffers and streams of their own: a synchronous call drains
// the slots above before it returns, and an asynchronous stage may still be in flight then.  Two, so that one stage's
// transfer overlaps the next one's kernels.
constexpr int NASYNC = 2;
struct AsyncSlot : SlotBase {
    DevBuf io;                             // the encode's dense output slots, or the decode's staged source
    DevBuf frames;                         // an LZ4Stream encode's frames, back to back, before they land
};
// The context's device cells that carry state from one pipeline stage to the next: the running output offset behind each
// slot's stage (run_host's packed decode into device memory, run_async's packed stages), the asynchronous LZ4Stream
// decode's failure flag, each asynchronous slot's device header walk.  The asynchronous cells are serialised by async_done.
struct Carry { int64_t host[NSLOT], async[NASYNC]; int failed; int64_t walk[NASYNC][STREAM_WALK_CELLS]; };
// The page-locked metadata of one asynchronous call, which the device reads after the call has returned: taken again once
// `done`, recorded behind the call, has fired.
struct MetaBlock { PinBuf buf; cudaEvent_t done = nullptr; bool used = false; };

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
// An asynchronous stage's device block (AsyncSlot::meta) holds every kind's: the arrays, a Wrap's or an Unwrap's
// WrapScratch at WRAP_META_OFFSET * m, then a packed form's "fits" flag (async_fits).
// The packet view (WrapScratch) of a stage of m blocks in its device block.
WrapScratch packet_view(void* meta, int32_t m) { return wrap_scratch_at((uint8_t*)meta + WRAP_META_OFFSET * (size_t)m, m); }
// The bytes of a stage's Meta h copied up: the four arrays the kernels read, and aux (stored lengths, lift bounds).
size_t meta_up_bytes(const Meta& h, bool aux) { return (size_t)((uint8_t*)(aux ? h.out : h.aux) - (uint8_t*)h.so); }
size_t async_meta_bytes(int32_t m) { return (size_t)m * WRAP_META_BYTES + sizeof(int64_t); }
int* async_fits(void* meta, int32_t m) { return (int*)((uint8_t*)meta + (size_t)m * WRAP_META_BYTES); }

// The operations of the batch codec.
enum class Op { ENCODE_FAST, ENCODE_HC, DECODE_KNOWN, DECODE_UNKNOWN, MEASURE_KNOWN, MEASURE_UNKNOWN };
constexpr Op encode_op(bool hc) { return hc ? Op::ENCODE_HC : Op::ENCODE_FAST; }
constexpr bool is_encode(Op op) { return op == Op::ENCODE_FAST || op == Op::ENCODE_HC; }
constexpr bool is_decode(Op op) { return op == Op::DECODE_KNOWN || op == Op::DECODE_UNKNOWN; }
constexpr bool is_measure(Op op) { return op == Op::MEASURE_KNOWN || op == Op::MEASURE_UNKNOWN; }

// What a stage of the host pipeline (run_host) runs on its chunk.
enum class Stage {
    CODEC,            // the operation (run_device)
    STREAM_ENCODE,    // the encode, then the chunks' LZ4Stream frames (lz4_stream.cuh, write_frames) in place of the
                      // compaction: APPEND lands the frames, out_off[i] = where frame i starts; asynchronously, the landing
                      // kernel does, keeping only the total
    WRAP_ENCODE,      // prep -> the encode -> finish (run_wrap, lz4_wrap.cuh): dst_cap[i] = the packet's capacity,
                      // src_len[i] + 8; the slot then holds whole packets, which land like the blocks of an encode
    FRAMED_DECODE,    // the known-size decode of LZ4Stream chunks or Unwrap packets: stored[i] != 0 marks a stored one, whose
                      // payload the stored-copy step copies while the decoder gets the neutral entry (src_len 0, dst_cap 0);
                      // in host memory it lands like a decoded block of dst_cap[i] bytes
    PLACED_DECODE,    // the packed unknown-size decode into device memory, its output offset carried across the stages
    UNWRAP,           // asynchronous calls only: Unwrap packets whose headers are read on the device (run_unwrap) into device
                      // memory, into the caller's slots, or packed (dst_off == nullptr) and placed like PLACED_DECODE
};

}  // namespace

struct lz4b200_ctx {
    int device = 0;
    DeviceInfo dev{};
    uint32_t* counters = nullptr;          // NCOUNTER words of the ring, then NCAPTURED sets of the capture pool
    int next_counter = 0;
    int next_captured = 0;                 // capture pool sets handed out
    SharedBuf hc_arena, compact_tmp;
    SharedBuf packed_caps;                 // lz4b200_decode_batch_packed: per-block capacities + the "fits" flag (serialised like compact_tmp)
    SharedBuf wrap_tmp;                    // the device Wrap / Unwrap calls: the codec's view of the packets (serialised like compact_tmp)
    std::vector<void*> retired;            // shared scratch a graph may still reference: freed by lz4b200_destroy
    Chain hc_done;                         // the HC state arena is shared: HC launches are chained through this event
    Chain compact_done;                    // likewise compact_tmp, packed_caps and wrap_tmp (DeviceCall)
    Chain async_done;                      // likewise the asynchronous calls' stage buffers, carry cells and streams (run_async)
    cudaEvent_t entry = nullptr;           // mixed-memory batches: recorded on the caller's stream, waited on by every slot
    Carry* carry = nullptr;                // device memory
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
    AsyncSlot aslot[NASYNC];
    std::vector<std::unique_ptr<MetaBlock>> meta_pool;    // the asynchronous calls' metadata (take_meta)
    int64_t launches = 0;
    std::mutex mu;

    // fours: [block counter, decoder pick, two more counters].  A captured call keeps its set for every replay: it takes one
    // of the capture pool, which admit() has checked is not used up.
    uint32_t* counter(const Capture& cap = {})
    {
        if (cap.on) return counters + NCOUNTER + 4 * next_captured++;
        uint32_t* c = counters + next_counter; next_counter = (next_counter + 4) % NCOUNTER; return c;
    }
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

// Whether `st` is capturing.  Every call that takes a stream asks this before it takes any scratch or synchronises.
int capture_of(cudaStream_t st, Capture* cap)
{
    cudaStreamCaptureStatus s = cudaStreamCaptureStatusNone;
    CU(cudaStreamGetCaptureInfo(st, &s, &cap->id));
    cap->on = s != cudaStreamCaptureStatusNone;
    return LZ4B200_OK;
}

// The calls that synchronise with the host, and the asynchronous calls, whose metadata is host data a graph would have to
// keep alive, refuse a capturing stream before any CUDA work, which leaves the caller's capture valid.
int refuse_capture(void* stream, const char* what, bool synchronises = true)
{
    Capture cap;
    int rc = capture_of((cudaStream_t)stream, &cap); if (rc) return rc;
    return cap.on ? fail(LZ4B200_E_ARG, std::string(what) + (synchronises ? " synchronises with the host: it" : "") +
                                            " cannot be enqueued on a capturing stream")
                  : LZ4B200_OK;
}

// What a device call takes: counter sets of the capture pool when captured (0 or 1), and bytes of the scan scratch, the
// packed calls' capacities + "fits" flag, the packet view and the HC arena.  need_of: a call family's need at n blocks
// (pieces: the ones it uses), for the calls and lz4b200_reserve alike; the HC arena under the current options, for
// hc_large blocks above 64 KiB (-1 = not known).
struct Need { int counters = 0; size_t scan = 0, caps = 0, wrap = 0, hc = 0; };
enum : unsigned { SCAN = 1, CAPS = 2, WRAP = 4, HC = 8 };
Need need_of(const lz4b200_ctx* c, int32_t n, unsigned pieces, int counters, int32_t hc_large = -1)
{
    Need d{counters};
    if (pieces & SCAN) d.scan = compact_tmp_bytes(n);
    if (pieces & CAPS) d.caps = sizeof(int32_t) * ((size_t)n + 1);
    if (pieces & WRAP) d.wrap = (size_t)n * WRAP_SCRATCH_BYTES;
    if (pieces & HC)
        d.hc = c->hc_kernel < 0 ? hc_auto_scratch_bytes(n, hc_large, c->dev)
             : c->hc_kernel ? hcw_scratch_bytes(n, hc_large, c->hc_kernel, c->hc_warps_per_sm, c->dev)
                            : hc_scratch_bytes((int)std::min<int64_t>(c->hc_concurrency, std::max(n, 1)));
    return d;
}

bool covers(const lz4b200_ctx* c, const Need& d)
{
    return d.scan <= c->compact_tmp.cap && d.caps <= c->packed_caps.cap && d.wrap <= c->wrap_tmp.cap && d.hc <= c->hc_arena.cap;
}

// Grows the shared scratch to cover `d`, behind one cudaDeviceSynchronize, since an earlier call may still be using it.
// Eager calls and lz4b200_reserve only.
int grow_scratch(lz4b200_ctx* c, const Need& d)
{
    if (covers(c, d)) return LZ4B200_OK;
    CU(cudaDeviceSynchronize());
    CU(c->compact_tmp.grow(d.scan, c->retired)); CU(c->packed_caps.grow(d.caps, c->retired));
    CU(c->wrap_tmp.grow(d.wrap, c->retired)); CU(c->hc_arena.grow(d.hc, c->retired));
    return LZ4B200_OK;
}

// A captured call never allocates, frees or synchronises: it enqueues nothing unless the scratch it needs is already there
// at its size (lz4b200_reserve grows it) and the capture pool has the counter sets it takes.  The buffers it references
// are then held for the graph.
int admit(lz4b200_ctx* c, const Need& d)
{
    if (!covers(c, d))
        return fail(LZ4B200_E_ARG, "the context's scratch is too small to capture this call: call lz4b200_reserve(ctx, n_blocks, "
                                   "high_compression) before capturing");
    if (c->next_captured + d.counters > NCAPTURED)
        return fail(LZ4B200_E_ARG, "the context's " + std::to_string(NCAPTURED) + " counter sets for captured calls are used up");
    if (d.scan) c->compact_tmp.held = true;
    if (d.caps) c->packed_caps.held = true;
    if (d.wrap) c->wrap_tmp.held = true;
    if (d.hc) c->hc_arena.held = true;
    return LZ4B200_OK;
}

// The way into every device-memory call, after its argument checks: the context's lock and device; then enter(need) admits
// a captured call or grows an eager one's scratch and, if it takes call scratch (compact_tmp, packed_caps, wrap_tmp: shared
// by the device calls on every stream), orders the stream behind the last such call.  Such a call closes with done() once
// its launches are in; one that fails records nothing, so a failed captured call leaves no event node in the graph.
struct DeviceCall : CallGuard {
    lz4b200_ctx* c; cudaStream_t st; Capture cap;
    DeviceCall(lz4b200_ctx* c, void* stream) : CallGuard(c), c(c), st((cudaStream_t)stream) {}
    int enter(const Need& d)
    {
        int rc = capture_of(st, &cap); if (rc) return rc;
        rc = cap.on ? admit(c, d) : grow_scratch(c, d); if (rc) return rc;
        if (d.scan || d.caps || d.wrap) CU(c->compact_done.wait(st, cap));
        return LZ4B200_OK;
    }
    int done() { CU(c->compact_done.record(st, cap)); return LZ4B200_OK; }
};

int launched(cudaError_t e, const char* what) { return e == cudaSuccess ? LZ4B200_OK : cuda_fail(e, what); }

// The lengths of a batch of blocks or packets (unit) whose arrays are on the host: src_len and, when given, dst_cap.
int check_lengths(const int32_t* src_len, const int32_t* dst_cap, int32_t n, const char* unit)
{
    for (int32_t i = 0; i < n; i++)
        if (src_len[i] < 0 || (dst_cap && dst_cap[i] < 0)) return fail(LZ4B200_E_ARG, std::string("negative ") + unit + " length");
    return LZ4B200_OK;
}

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

// hc_large: blocks above 64 KiB in an HC batch (-1 = not known: a device-memory batch).  A captured call (cap) has been
// admitted with the arena and the counter set it takes.
int run_device(lz4b200_ctx* c, const BatchArgs& a, Op op, cudaStream_t st, int lanes = 0, int32_t hc_large = -1, const Capture& cap = {})
{
    if (!lanes) lanes = c->pinned_lanes();
    cudaError_t e = cudaSuccess;
    switch (op) {
    case Op::ENCODE_FAST: e = launch_encode_fast(a, c->counter(cap), c->encode_ctas_per_sm, c->encode_tune, c->encode_variant, c->dev, st, &c->launches); break;
    case Op::ENCODE_HC: {
        const int conc = (int)std::min<int64_t>(c->hc_concurrency, std::max(a.n_blocks, 1));
        if (!cap.on) { int rc = grow_scratch(c, need_of(c, a.n_blocks, HC, 0, hc_large)); if (rc) return rc; }
        // one arena per context: an HC launch may not overlap the previous one, whatever stream it was given
        CU(c->hc_done.wait(st, cap));
        uint32_t* counter = c->counter(cap);
        e = c->hc_kernel < 0 ? launch_encode_hc_auto(a, c->hc_arena.p, hc_large, counter, c->dev, st, &c->launches)
          : c->hc_kernel ? launch_encode_hcw(a, c->hc_arena.p, c->hc_kernel, c->hc_warps_per_sm, hc_large, counter, c->dev, st, &c->launches)
                              : launch_encode_hc(a, c->hc_arena.p, conc, counter, c->dev, st, &c->launches);
        if (e == cudaSuccess) e = c->hc_done.record(st, cap);
        break;
    }
    case Op::DECODE_KNOWN:
    case Op::DECODE_UNKNOWN: e = launch_decode(a, op == Op::DECODE_KNOWN, lanes, c->counter(cap), c->dev, st, &c->launches); break;
    case Op::MEASURE_KNOWN:
    case Op::MEASURE_UNKNOWN: e = launch_measure(a, op == Op::MEASURE_KNOWN, c->dev, st, &c->launches); break;
    }
    return launched(e, "kernel launch");
}

// A Wrap of the batch a into whole packets: prep (each payload behind its header's place, capacity = its input length,
// LZ4Codec.cs:518-523) -> the batch codec, unchanged, on the codec's view w -> finish (the headers, the stored inputs,
// out_len = the packet sizes).
int run_wrap(lz4b200_ctx* c, const BatchArgs& a, const WrapScratch& w, Op op, cudaStream_t st, int32_t hc_large, const Capture& cap = {})
{
    int rc = launched(launch_wrap_prep(a, w, st, &c->launches), "wrap prep launch"); if (rc) return rc;
    const BatchArgs enc{a.src, a.src_off, w.len, a.dst, w.off, w.cap, w.res, a.n_blocks};
    rc = run_device(c, enc, op, st, 0, hc_large, cap); if (rc) return rc;
    return launched(launch_wrap_finish(a, w, st, &c->launches), "wrap finish launch");
}

// The placement of a packed decode (lz4_packed.cuh): the sizes scanned into `off` (scan: the scan's scratch), then each
// block's capacity (its size + room) into caps, and the "fits" flag against total_cap.  A pipeline stage places behind the
// previous one: it waits on `after`, starts from the running total in `base` (null for the first stage), leaves its
// absolute offsets in abs_off and the running total in `total`, and records `placed` once placed.  A batch placed in one
// piece leaves those null.
struct Placement {
    int64_t* off; void* scan; size_t scan_bytes;
    int64_t total_cap; int32_t room; int32_t* caps; int* fits;
    cudaEvent_t after = nullptr; const int64_t* base = nullptr; int64_t* abs_off = nullptr; int64_t* total = nullptr;
    cudaEvent_t placed = nullptr;
};

cudaError_t place(lz4b200_ctx* c, const int32_t* size, int32_t n, const Placement& p, cudaStream_t st)
{
    cudaError_t e = launch_compact(nullptr, nullptr, size, nullptr, p.off, n, p.scan, p.scan_bytes, c->dev, st, &c->launches);
    if (e == cudaSuccess && p.after) e = cudaStreamWaitEvent(st, p.after, 0);
    if (e == cudaSuccess)
        e = launch_packed_prep(size, p.off, n, p.total_cap, p.room, p.caps, p.fits, st, &c->launches, p.base, p.abs_off, p.total);
    if (e == cudaSuccess && p.placed) e = cudaEventRecord(p.placed, st);
    return e;
}

// A pipeline stage's placement on slot sl (metadata d), behind the previous stage's (prev: its slot and the carry cell
// `base` it leaves; none for the first stage); it leaves its running total in `total` and records sl's `carried`.
Placement chained_placement(SlotBase& sl, const Meta& d, int* fits, int64_t total_cap, const SlotBase* prev, const int64_t* base, int64_t* total)
{
    return Placement{(int64_t*)sl.offs.p, sl.scan.p, sl.scan.cap, total_cap, 0, d.dc, fits, prev ? prev->carried : nullptr,
                     prev ? base : nullptr, d.dof, total, sl.carried};
}

// An Unwrap of the packets of a (src / src_off / src_len; outputs at dst + dst_off, capacities dst_cap, null = no limit):
// prep (each header, read on the device: a decode entry for a compressed packet, a neutral one for a stored or rejected
// packet) -> [the packed forms: the placement of the sizes the prep left in out_len, which writes the decode's capacities
// and the "fits" flag that both the decode and the finish run behind] -> the known-size decode -> finish (the stored
// copies, out_len = bytes restored or the packet's status).  The counterpart of run_wrap, for the device calls and the
// asynchronous stages alike.
int run_unwrap(lz4b200_ctx* c, const BatchArgs& a, const WrapScratch& w, cudaStream_t st, const Capture& cap = {},
               const Placement* placed = nullptr)
{
    int rc = launched(launch_unwrap_prep(a, w, st, &c->launches), "unwrap prep launch"); if (rc) return rc;
    if (placed) { rc = launched(place(c, a.out_len, a.n_blocks, *placed, st), "unwrap placement launch"); if (rc) return rc; }
    // the compressed packets, known size (LZ4Codec.cs:595); stored and rejected ones are neutral entries
    const BatchArgs dec{a.src, w.off, w.len, a.dst, a.dst_off, placed ? placed->caps : w.cap, w.res, a.n_blocks};
    const int* fits = placed ? placed->fits : nullptr;
    rc = launched(launch_decode(dec, true, c->pinned_lanes(), c->counter(cap), c->dev, st, &c->launches, fits), "unwrap decode launch");
    if (rc) return rc;
    return launched(launch_unwrap_finish(a, w, fits, st, &c->launches), "unwrap finish launch");
}

// The packed unknown-size decode of a, whose dst_off and dst_cap are the placement's abs_off (or off) and caps: measure
// (no capacity) -> place the sizes, with the room of an unknown-size decode -> the decode behind the "fits" flag, whose
// decoders leave at once when the total does not fit, so out_len keeps the measured sizes and dst is untouched.
int run_placed_decode(lz4b200_ctx* c, const BatchArgs& a, Placement p, cudaStream_t st, const Capture& cap = {})
{
    p.room = PACKED_ROOM_UNKNOWN;
    BatchArgs sizes = a; sizes.dst_cap = nullptr;
    cudaError_t e = launch_measure(sizes, false, c->dev, st, &c->launches);
    if (e == cudaSuccess) e = place(c, a.out_len, a.n_blocks, p, st);
    if (e == cudaSuccess) e = launch_decode(a, false, c->pinned_lanes(), c->counter(cap), c->dev, st, &c->launches, p.fits);
    return launched(e, "packed measure / placement / decode launch");
}

// What a stage of run_host or run_async runs on its blocks a (lanes, hc_large: its decoder and HC arena, stage_lanes and
// stage_hc_large): w is the stage's packet view (WRAP_ENCODE, UNWRAP), placed its placement (PLACED_DECODE, a packed
// UNWRAP) and stored a FRAMED_DECODE's stored lengths.
int run_stage(lz4b200_ctx* c, Stage kind, Op op, const BatchArgs& a, int lanes, int32_t hc_large, const WrapScratch& w,
              const Placement* placed, const int32_t* stored, cudaStream_t st)
{
    switch (kind) {
    case Stage::CODEC:
    case Stage::STREAM_ENCODE: return run_device(c, a, op, st, lanes, hc_large);
    case Stage::WRAP_ENCODE: return run_wrap(c, a, w, op, st, hc_large);
    case Stage::FRAMED_DECODE: {
        int rc = run_device(c, a, op, st, lanes); if (rc) return rc;
        return launched(launch_stream_stored(a, stored, st, &c->launches), "stored copy launch");
    }
    case Stage::PLACED_DECODE: return run_placed_decode(c, a, *placed, st);
    case Stage::UNWRAP: return run_unwrap(c, a, w, st, {}, placed);
    }
    return fail(LZ4B200_E_ARG, "unknown stage kind");
}

// The LZ4Stream frames of an encoded STREAM_ENCODE stage a, back to back: the frame sizes into frame_len, their scan into
// offs (offs[m] = the stage's bytes), then each frame at frames + offs[i].  In place of the compaction, in run_host and
// run_async alike.
cudaError_t write_frames(lz4b200_ctx* c, const BatchArgs& a, bool hc, int32_t* frame_len, int64_t* offs, void* scan,
                         size_t scan_bytes, uint8_t* frames, cudaStream_t st)
{
    cudaError_t e = launch_stream_frame_size(a, frame_len, st, &c->launches);
    if (e == cudaSuccess) e = launch_compact(nullptr, nullptr, frame_len, nullptr, offs, a.n_blocks, scan, scan_bytes, c->dev, st, &c->launches);
    if (e == cudaSuccess) e = launch_stream_frame(a, hc, frames, offs, st, &c->launches);
    return e;
}

// ---- the stage plan of the host pipeline, shared by run_host and the asynchronous calls (run_async) ------------------
// A stage [b0, b1) is weighed by the bytes it stages: src_len[i] when count_src, plus dst_cap[i] when dst_cap is given
// (not for a destination already on the device, nor for the measure pass).  Blocks join it while it stays within
// host_chunk_bytes; it takes at least one.
int32_t stage_end(const lz4b200_ctx* c, const int32_t* src_len, const int32_t* dst_cap, int32_t b0, int32_t n, bool count_src)
{
    int64_t bytes = 0; int32_t b1 = b0;
    while (b1 < n) {
        const int64_t w = (count_src ? (int64_t)src_len[b1] : 0) + (dst_cap ? dst_cap[b1] : 0);
        if (b1 > b0 && bytes + w > (int64_t)c->host_chunk_bytes) break;
        bytes += w; b1++;
    }
    return b1;
}

// Host bytes of a stage's Meta of m blocks (packed_off included).
size_t meta_host_bytes(int32_t m) { return (size_t)m * META_BYTES + sizeof(int64_t) * (size_t)(m + 2); }

// What fill_stage leaves besides the metadata: the source range the stage stages, [slo, shi) (0, 0 when the source is on
// the device), and the bytes of its dense output slots (0 when the destination is).
struct StageSpan { int64_t slo = 0, shi = 0, dsum = 0; };

// The stage's metadata in h: source offsets relative to the staged range, destination offsets (dense slots, or the
// caller's own when the destination is on the device; 0 for a placed decode, which places on the device), lengths and
// capacities; a framed decode's stored entries (stored != null) become neutral, their lengths in aux.
StageSpan fill_stage(const Meta& h, int32_t b0, int32_t b1, const int64_t* src_off, const int32_t* src_len, const int64_t* dst_off,
                     const int32_t* dst_cap, bool src_dev, bool dst_dev, bool measure, bool placed, const uint8_t* stored)
{
    StageSpan sp;
    const int32_t m = b1 - b0;
    if (!src_dev) {
        sp.slo = INT64_MAX; sp.shi = INT64_MIN;
        for (int32_t i = b0; i < b1; i++) { sp.slo = std::min(sp.slo, src_off[i]); sp.shi = std::max(sp.shi, src_off[i] + src_len[i]); }
    }
    for (int32_t i = 0; i < m; i++) {
        h.so[i] = src_off[b0 + i] - sp.slo;
        if (dst_dev) h.dof[i] = placed ? 0 : dst_off[b0 + i];
        else { h.dof[i] = sp.dsum; sp.dsum += measure ? 0 : dst_cap[b0 + i]; }
        h.sl[i] = src_len[b0 + i]; h.dc[i] = dst_cap ? dst_cap[b0 + i] : INT32_MAX;
        if (stored) {
            const bool st = stored[b0 + i] != 0;
            h.aux[i] = st ? h.sl[i] : 0;
            if (st) h.sl[i] = h.dc[i] = 0;
        }
    }
    return sp;
}

// The decoder of a decode stage, from its compression ratio (0: the context's pinned choice, or not a decode, or a placed
// stage, whose decoded sizes are known on the device only: dst_cap == nullptr).
int stage_lanes(const lz4b200_ctx* c, Op op, const int32_t* src_len, const int32_t* dst_cap, int32_t b0, int32_t b1)
{
    if (!is_decode(op) || !c->decode_lanes_auto || !dst_cap) return 0;
    double cs = 0, rs = 0;
    for (int32_t i = b0; i < b1; i++) { cs += src_len[i]; rs += dst_cap[i]; }
    return lanes_for_ratio(rs > 0 ? cs / rs : 1.0, b1 - b0, c->dev);
}

// The blocks above 64 KiB of an HC encode stage (they size the HC arena).
int32_t stage_hc_large(Op op, const int32_t* src_len, int32_t b0, int32_t b1)
{
    int32_t k = 0;
    if (op == Op::ENCODE_HC) for (int32_t i = b0; i < b1; i++) k += src_len[i] > 65536;
    return k;
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
    int rc = check_lengths(src_len, dst_cap, n, "block"); if (rc) return rc;
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
        const int32_t b1 = stage_end(c, src_len, measure || dst_dev ? nullptr : dst_cap, b0, n, !src_dev);
        const int s = k % NSLOT; k++;
        rc = retire(s); if (rc) return rc;
        Slot& sl = c->slot[s];
        const int32_t m = b1 - b0;
        const Mode mode = measure || dst_dev ? NONE : !dst_off ? APPEND : m <= 8 ? PER_BLOCK : op == Op::DECODE_KNOWN ? RUNS : SCATTER;
        CU(sl.meta.reserve((size_t)m * (kind == Stage::WRAP_ENCODE ? WRAP_META_BYTES : META_BYTES) + (placed ? sizeof(int64_t) : 0)));
        CU(sl.hmeta.reserve(meta_host_bytes(m)));
        const Meta h(sl.hmeta.p, m), d(sl.meta.p, m);
        const StageSpan sp = fill_stage(h, b0, b1, src_off, src_len, dst_off, dst_cap, src_dev, dst_dev, measure, placed,
                                        framed ? stored : nullptr);
        const int64_t slo = sp.slo, dsum = sp.dsum;
        const size_t sbytes = (size_t)(sp.shi - slo);
        if (!src_dev) CU(sl.src.reserve(sbytes + 64));
        if (!dst_dev) CU(sl.dst.reserve((size_t)dsum + 64));
        CU(cudaMemcpyAsync(sl.meta.p, sl.hmeta.p, meta_up_bytes(h, framed), cudaMemcpyHostToDevice, sl.stream));
        if (sbytes) {
            const uint8_t* from = src + slo;
            if (src_pageable && m > 8) { CU(sl.hsrc.reserve(sbytes)); par_memcpy(sl.hsrc.p, from, sbytes); from = (const uint8_t*)sl.hsrc.p; }
            CU(cudaMemcpyAsync(sl.src.p, from, sbytes, cudaMemcpyHostToDevice, sl.stream));
        }
        const BatchArgs a{src_dev ? src : (const uint8_t*)sl.src.p, d.so, d.sl, dst_dev ? dst : (uint8_t*)sl.dst.p, d.dof, d.dc, d.out, m};
        Placement pl{};
        if (placed) {
            // behind the previous stage's placement; the stage's "fits" flag lives behind its arrays (Meta)
            CU(sl.offs.reserve(sizeof(int64_t) * (size_t)(m + 1))); CU(sl.scan.reserve(compact_tmp_bytes(m)));
            const int prev = (s + NSLOT - 1) % NSLOT;
            pl = chained_placement(sl, d, (int*)d.off, dst_total_cap, b0 > 0 ? &c->slot[prev] : nullptr, &c->carry->host[prev],
                                   &c->carry->host[s]);
        }
        rc = run_stage(c, kind, op, a, stage_lanes(c, op, src_len, dst_cap, b0, b1), stage_hc_large(op, src_len, b0, b1),
                       packet_view(sl.meta.p, m), placed ? &pl : nullptr, d.aux, sl.stream);
        if (rc) return rc;
        if (placed) {
            CU(cudaMemcpyAsync(h.dof, d.dof, sizeof(int64_t) * (size_t)m, cudaMemcpyDeviceToHost, sl.stream));
            CU(cudaMemcpyAsync(h.off, &c->carry->host[s], sizeof(int64_t), cudaMemcpyDeviceToHost, sl.stream));
        }
        if (mode >= SCATTER) {
            // the outputs back to back: compacted, or an LZ4Stream encode's frames (sizes -> scan -> headers + payloads)
            const bool frames = kind == Stage::STREAM_ENCODE;
            CU(sl.packed.reserve((size_t)dsum + (frames ? (size_t)m * STREAM_HEADER_MAX : 0) + 64));
            CU(sl.offs.reserve(sizeof(int64_t) * (size_t)(m + 1))); CU(sl.scan.reserve(compact_tmp_bytes(m)));
            uint8_t* packed = (uint8_t*)sl.packed.p;
            int64_t* offs = (int64_t*)sl.offs.p;
            const cudaError_t e =
                frames ? write_frames(c, a, op == Op::ENCODE_HC, d.aux, offs, sl.scan.p, sl.scan.cap, packed, sl.stream)
                       : launch_compact(a.dst, a.dst_off, a.out_len, packed, offs, m, sl.scan.p, sl.scan.cap, c->dev, sl.stream, &c->launches);
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
    for (int i = 0; i < NSLOT; i++) { rc = retire((k + i) % NSLOT); if (rc) return rc; }
    if (out_off) out_off[n] = written;
    return LZ4B200_OK;
}

// The side of a mixed-memory call that must be device memory is memory of the context's device (plain or managed); the
// side that must be host memory is not device memory (pageable, page-locked or managed host memory all copy).
int check_side(const lz4b200_ctx* c, const void* p, bool device, const char* what)
{
    const cudaPointerAttributes a = pointer_attributes(p);
    const bool on_device = a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
    if (device && !(on_device && a.device == c->device))
        return fail(LZ4B200_E_ARG, std::string(what) + " must be device memory of the context's GPU");
    if (!device && a.type == cudaMemoryTypeDevice) return fail(LZ4B200_E_ARG, std::string(what) + " must be host memory");
    return LZ4B200_OK;
}

// ---- the asynchronous calls between device memory and page-locked host memory (run_async) ---------------------------
// The address at which the device reaches p, for a buffer the device reads or writes after an asynchronous call has
// returned: page-locked host memory with a device address (cudaHostAlloc / cudaMallocHost, torch pin_memory(), a
// lz4b200_host_register'd range), or, when `device_ok`, device memory of the context's GPU.
int device_address(const lz4b200_ctx* c, const void* p, bool device_ok, const char* what, void** at)
{
    const cudaPointerAttributes a = pointer_attributes(p);
    if (a.type == cudaMemoryTypeHost && a.devicePointer) { *at = a.devicePointer; return LZ4B200_OK; }
    if (device_ok && (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == c->device) {
        *at = const_cast<void*>(p);
        return LZ4B200_OK;
    }
    return fail(LZ4B200_E_ARG, std::string(what) + (device_ok ? " must be device memory of the context's GPU or page-locked host memory"
                                                              : " must be page-locked host memory the device can address"));
}

// A page-locked metadata block of at least `bytes` whose last call the device has passed (cudaEventQuery, never waited
// on).  The pool grows when none is free; a free block too small is grown (which may synchronise, as a growth may).
int take_meta(lz4b200_ctx* c, size_t bytes, MetaBlock** out)
{
    MetaBlock *fit = nullptr, *small = nullptr;
    for (auto& b : c->meta_pool) {
        if (b->used) {
            const cudaError_t q = cudaEventQuery(b->done);
            if (q == cudaErrorNotReady) continue;
            if (q != cudaSuccess) return cuda_fail(q, "cudaEventQuery");
            b->used = false;
        }
        if (b->buf.cap >= bytes) { if (!fit || b->buf.cap < fit->buf.cap) fit = b.get(); }
        else small = b.get();
    }
    if (!fit) {
        if (!small) {
            c->meta_pool.emplace_back(new MetaBlock());
            small = c->meta_pool.back().get();
            CU(cudaEventCreateWithFlags(&small->done, cudaEventDisableTiming));
        }
        CU(small->buf.reserve(bytes));
        fit = small;
    }
    fit->used = true;
    *out = fit;
    return LZ4B200_OK;
}

// The LZ4Stream calls run the pipeline over at most this many chunks at a time: it bounds the host metadata by chunk
// count (tiny blocks would otherwise need gigabytes of it), while a call covers many pipeline stages.  An asynchronous
// encode stage takes at most this many chunks, which bounds its device metadata the same way.
constexpr int64_t STREAM_RUN_CHUNKS = 1 << 20;

// The decode entries of an LZ4Stream of n bytes at s, from its header walk (stream_walk): one per non-empty chunk, with
// its payload offset, compLen, output offset, rawLen and stored flag -- the header's flag: a compressed chunk may have
// compLen == rawLen (LZ4Stream.cs:288).  Returns the decoded size or LZ4B200_E_FORMAT.
struct StreamEntries { std::vector<int64_t> so, dof; std::vector<int32_t> len, raw; std::vector<uint8_t> stored; };
int64_t stream_entries(const uint8_t* s, int64_t n, StreamEntries* e)
{
    std::vector<StreamChunk> chunks;
    const int64_t total = stream_walk(s, n, &chunks);
    if (total < 0) return total;
    int64_t pos = 0;
    for (const StreamChunk& k : chunks) {
        if (k.raw > 0) {
            e->so.push_back(k.payload); e->len.push_back(k.stored); e->dof.push_back(pos); e->raw.push_back(k.raw);
            e->stored.push_back(!k.compressed);
        }
        pos += k.raw;
    }
    return total;
}

// Where the blocks of an asynchronous call's stages come from.
enum class Source {
    DEVICE,    // device memory, read in place, with host entries: the packed encodes
    COPIED,    // page-locked host memory copied up a stage at a time, with host entries: the decodes
    CUT,       // device memory, the entries cut on the device (stream_cut_one): the LZ4Stream encode
    LIFTED,    // page-locked host memory lifted by offsets read on the device (lz4_lift.cuh): the _at decode and Unwrap
    WALKED,    // page-locked host memory, its headers walked on the device (stream_walk_stage): the _at LZ4Stream decode
};

// One asynchronous call: what its stages run (kind, op), where their blocks come from, the caller's arrays, and the few
// fields of the LZ4Stream and lifted calls, in that order.  out_off is an LZ4Stream call's out_size.
struct AsyncCall {
    Stage kind; Op op; Source from;
    const uint8_t* src = nullptr; const int64_t* src_off = nullptr; const int32_t* src_len = nullptr;
    uint8_t* dst = nullptr; const int64_t* dst_off = nullptr; const int32_t* dst_cap = nullptr;
    int32_t* out_len = nullptr; int32_t n = 0; int64_t* out_off = nullptr; int64_t dst_total_cap = 0;
    int64_t src_cap = 0;                   // LIFTED, WALKED: the bytes of src that may be read
    const int64_t* src_size = nullptr;     // WALKED: where the stream's size S is
    int64_t stream_len = 0;                // CUT, and COPIED into FRAMED_DECODE: the stream's length
    int32_t block_size = 0;                // CUT, WALKED: the chunk size
    std::vector<int32_t> bound;            // LIFTED: each block's bound, by which the stages are cut and their slots sized
    const uint8_t* stored = nullptr;       // COPIED into FRAMED_DECODE: the entries' stored flags
    int64_t total = 0;                     //   and the decoded size
    // the packed decodes, whose stages place their blocks on the device (lz4_packed.cuh)
    bool placed() const { return kind == Stage::PLACED_DECODE || (kind == Stage::UNWRAP && !dst_off); }
};

// A lift stage's metadata: dst_off / dst_cap as the caller gave them, each block's slot (so[i], and its prefix in off[0..m])
// and its bound (aux); the spans are written on the device.  sp.shi = the stage's staging bytes.
StageSpan fill_lift(const Meta& h, int32_t b0, int32_t b1, const int32_t* bound, const int64_t* dst_off, const int32_t* dst_cap)
{
    StageSpan sp;
    for (int32_t i = 0; i < b1 - b0; i++) {
        h.off[i] = h.so[i] = sp.shi;
        h.dof[i] = dst_off[b0 + i]; h.sl[i] = 0; h.dc[i] = dst_cap[b0 + i]; h.aux[i] = bound[b0 + i];
        sp.shi += lift_slot_bytes(bound[b0 + i]);
    }
    h.off[b1 - b0] = sp.shi;
    return sp;
}

// A walk stage's device scratch, in AsyncSlot::offs: the lift descriptor the walk writes (STREAM_WALK_LIFT_I64 int64, then
// the int32 bound), then the lift's entry for its one block (so, then sl and dc).
constexpr size_t WALK_OFFS_BYTES = sizeof(int64_t) * (STREAM_WALK_LIFT_I64 + 3);

// An asynchronous stage: blocks [b0, b1), their host metadata at `at` in the call's block; or chunks [first, first + b1).
struct Plan { int32_t b0, b1; size_t at; StageSpan sp; int64_t first; };

// The stage plan by blocks (DEVICE, COPIED, LIFTED), cut as run_host cuts it (stage_end; a lifted one by the bounds),
// each stage described in the call's metadata block (fill_stage, fill_lift).
int plan_blocks(lz4b200_ctx* c, const AsyncCall& a, std::vector<Plan>& plan, MetaBlock** blk)
{
    const bool enc = is_encode(a.op), lifted = a.from == Source::LIFTED;
    size_t bytes = 0;
    for (int32_t b0 = 0; b0 < a.n;) {
        const int32_t b1 = stage_end(c, lifted ? a.bound.data() : a.src_len, enc ? a.dst_cap : nullptr, b0, a.n, !enc);
        plan.push_back(Plan{b0, b1, bytes, {}, 0});
        bytes += (meta_host_bytes(b1 - b0) + 15) & ~(size_t)15;
        b0 = b1;
    }
    int rc = take_meta(c, bytes, blk); if (rc) return rc;
    for (Plan& p : plan) {
        const Meta h((uint8_t*)(*blk)->buf.p + p.at, p.b1 - p.b0);
        p.sp = lifted ? fill_lift(h, p.b0, p.b1, a.bound.data(), a.dst_off, a.dst_cap)
                      : fill_stage(h, p.b0, p.b1, a.src_off, a.src_len, a.dst_off, a.dst_cap, enc, !enc, false, a.placed(), a.stored);
    }
    return LZ4B200_OK;
}

// The stage plan by chunks (CUT, WALKED): the stream's chunks of block_size bytes (the encode's input, the walk's output
// capacity), `per` a stage (as many as host_chunk_bytes holds, 1 to STREAM_RUN_CHUNKS), at least one stage (a walk's first
// checks S).  An encode stage's span is its input; a walk stage's, the bytes its lift stages: *span_cap.
void plan_chunks(const lz4b200_ctx* c, const AsyncCall& a, std::vector<Plan>& plan, int64_t* span_cap)
{
    const bool walked = a.from == Source::WALKED;
    const int64_t bs = a.block_size, len = walked ? a.dst_total_cap : a.stream_len, chunks = len / bs + (len % bs != 0);
    // a walk stage's span (a header may take STREAM_WALK_HEADER_MAX bytes) must fit an int32: the walk's cap alone
    const int64_t frame = bs + STREAM_WALK_HEADER_MAX, cap = walked ? INT32_MAX / frame : STREAM_RUN_CHUNKS;
    const int64_t per = std::max<int64_t>(1, std::min<int64_t>({(int64_t)c->host_chunk_bytes / bs, STREAM_RUN_CHUNKS, cap}));
    // (the chunks' payloads add up to at most dst_total_cap bytes, which bounds a walk stage's span for a small output)
    if (walked) *span_cap = std::min<int64_t>({per * frame, per * STREAM_WALK_HEADER_MAX + a.dst_total_cap, INT32_MAX});
    for (int64_t k0 = 0; k0 == 0 || k0 < chunks; k0 += per) {
        const int32_t m = (int32_t)std::min(per, chunks - k0);
        StageSpan sp;
        if (walked) sp.shi = lift_slot_bytes((int32_t)*span_cap);
        else sp.dsum = std::min((int64_t)m * bs, len - k0 * bs);
        plan.push_back(Plan{0, m, 0, sp, k0});
    }
}

// The stages of an asynchronous call, enqueued on the context's NASYNC streams in turn, forked from `caller` and joined
// back to it; nothing is waited on unless a buffer must grow.  A stage runs as arrival (by source: its entries and bytes
// on the device; a lifted or walked stage's decoder is then picked on the device), its kind's sequence (run_stage, as in
// run_host: the encoders write AsyncSlot::io, the decoders dst in place) and departure (by kind): the packed encodes'
// scan and landing (lz4_land.cuh), or the LZ4Stream encode's frames and their landing, behind the running total the
// previous stage left in its carry cell; an LZ4Stream decode's failure flag (Carry::failed, cleared behind the previous
// call); the other decodes' results, after a lifted stage's rejections, with a packed stage's absolute offsets (placed
// behind the previous stage's from the same cells) and the last running total.  Behind the join, on `caller`, an
// LZ4Stream call writes its size, or its decoded size or status (stream_result, stream_walk_result), to out_off[0].
// Calls are chained through async_done; the call's metadata block is taken again once the caller's stream has passed it.
int run_async(lz4b200_ctx* c, const AsyncCall& a, cudaStream_t caller)
{
    const bool enc = is_encode(a.op), placed = a.placed(), framed = a.kind == Stage::FRAMED_DECODE;
    std::vector<Plan> plan;
    MetaBlock* blk = nullptr;
    int64_t span_cap = 0;
    if (a.from == Source::CUT || a.from == Source::WALKED) plan_chunks(c, a, plan, &span_cap);
    else if (int rc = plan_blocks(c, a, plan, &blk)) return rc;
    struct Sizes { size_t io = 0, frames = 0, meta = 0, offs = 0, scan = 0; } need[NASYNC];      // each slot's buffers, for its largest stage
    for (size_t k = 0; k < plan.size(); k++) {
        const Plan& p = plan[k];
        const int32_t m = p.b1 - p.b0;
        Sizes& nd = need[k % NASYNC];
        nd.io = std::max(nd.io, (size_t)(enc ? p.sp.dsum : p.sp.shi - p.sp.slo) + 64);
        if (a.from == Source::CUT) nd.frames = std::max(nd.frames, (size_t)p.sp.dsum + (size_t)m * STREAM_HEADER_MAX + 64);
        nd.meta = std::max(nd.meta, async_meta_bytes(m));
        if (enc || placed) { nd.offs = std::max(nd.offs, sizeof(int64_t) * (size_t)(m + 1)); nd.scan = std::max(nd.scan, compact_tmp_bytes(m)); }
        if (a.from == Source::LIFTED) nd.offs = std::max(nd.offs, sizeof(int64_t) * (size_t)(2 * m + 3));      // slot[0..m] | span[0..m+1]
        if (a.from == Source::WALKED) nd.offs = std::max(nd.offs, WALK_OFFS_BYTES);
    }
    // growth: an earlier call may still be using the buffers
    bool grow = false;
    for (int s = 0; s < NASYNC; s++) {
        const AsyncSlot& sl = c->aslot[s];
        grow |= need[s].io > sl.io.cap || need[s].frames > sl.frames.cap || need[s].meta > sl.meta.cap || need[s].offs > sl.offs.cap ||
                need[s].scan > sl.scan.cap;
    }
    if (grow) {
        CU(cudaDeviceSynchronize());
        for (int s = 0; s < NASYNC; s++) {
            AsyncSlot& sl = c->aslot[s];
            CU(sl.io.reserve(need[s].io)); CU(sl.frames.reserve(need[s].frames)); CU(sl.meta.reserve(need[s].meta));
            CU(sl.offs.reserve(need[s].offs)); CU(sl.scan.reserve(need[s].scan));
        }
    }
    const int used = (int)std::min<size_t>(plan.size(), NASYNC);
    Carry* carry = c->carry;
    auto stages = [&]() -> int {
        if (framed) {
            // the failure flag, cleared behind the context's previous asynchronous call (which may still read it)
            CU(c->async_done.wait(caller, Capture{}));
            CU(cudaMemsetAsync(&carry->failed, 0, sizeof(int), caller));
        }
        CU(cudaEventRecord(c->entry, caller));
        for (int s = 0; s < used; s++) {
            CU(cudaStreamWaitEvent(c->aslot[s].stream, c->entry, 0));
            CU(c->async_done.wait(c->aslot[s].stream, Capture{}));
        }
        for (size_t k = 0; k < plan.size(); k++) {
            const Plan& p = plan[k];
            const int s = (int)(k % NASYNC), prev = (s + NASYNC - 1) % NASYNC;
            AsyncSlot& sl = c->aslot[s];
            const int32_t m = p.b1 - p.b0;
            const Meta d(sl.meta.p, m);
            int64_t* offs = (int64_t*)sl.offs.p;
            int64_t* span = offs + m + 1;
            auto up = [&](bool aux) { const Meta h((uint8_t*)blk->buf.p + p.at, m);
                                      return cudaMemcpyAsync(sl.meta.p, h.so, meta_up_bytes(h, aux), cudaMemcpyHostToDevice, sl.stream); };
            int rc = LZ4B200_OK;
            switch (a.from) {
            case Source::DEVICE: CU(up(false)); break;
            case Source::COPIED:
                CU(up(framed));
                if (p.sp.shi != p.sp.slo)
                    CU(cudaMemcpyAsync(sl.io.p, a.src + p.sp.slo, (size_t)(p.sp.shi - p.sp.slo), cudaMemcpyHostToDevice, sl.stream));
                break;
            case Source::CUT:
                rc = launched(launch_stream_cut(p.first, m, a.block_size, a.stream_len, d.so, d.sl, d.dof, d.dc, sl.stream, &c->launches),
                              "stream chunk table launch");
                break;
            case Source::LIFTED:
                CU(up(true));
                // the slots, then the stage's offsets and src_off[n], wherever the caller's src_off lives
                CU(cudaMemcpyAsync(offs, Meta((uint8_t*)blk->buf.p + p.at, m).off, sizeof(int64_t) * (size_t)(m + 1), cudaMemcpyHostToDevice,
                                   sl.stream));
                CU(cudaMemcpyAsync(span, a.src_off + p.b0, sizeof(int64_t) * (size_t)(m + 1), cudaMemcpyDefault, sl.stream));
                CU(cudaMemcpyAsync(span + m + 1, a.src_off + a.n, sizeof(int64_t), cudaMemcpyDefault, sl.stream));
                rc = launched(launch_lift(a.src, a.src_cap, offs, span, m, p.sp.shi, d.aux, d.so, d.sl, d.dc, (uint8_t*)sl.io.p, c->dev,
                                          sl.stream, &c->launches), "lift launch");
                break;
            case Source::WALKED: {
                // behind the previous stage's walk only; the next stage's walk follows this one, not its lift or decode
                if (k > 0) CU(cudaStreamWaitEvent(sl.stream, c->aslot[prev].carried, 0));
                const StreamWalkStage w{a.src, a.src_cap, k == 0 ? a.src_size : nullptr, k > 0 ? carry->walk[prev] : nullptr,
                                        carry->walk[s], a.block_size, a.dst_total_cap, m, k + 1 == plan.size(), span_cap,
                                        d.so, d.dof, d.sl, d.dc, d.aux, offs};
                rc = launched(launch_stream_walk(w, sl.stream, &c->launches), "stream walk launch"); if (rc) return rc;
                CU(cudaEventRecord(sl.carried, sl.stream));
                if (m == 0) continue;
                // the stage's span, as the lift's one block
                int32_t* lifted = (int32_t*)(offs + STREAM_WALK_LIFT_I64 + 2);
                rc = launched(launch_lift(a.src, a.src_cap, offs, offs + 2, 1, p.sp.shi, (const int32_t*)(offs + STREAM_WALK_LIFT_I64),
                                          offs + STREAM_WALK_LIFT_I64 + 1, lifted, lifted + 1, (uint8_t*)sl.io.p, c->dev, sl.stream,
                                          &c->launches), "stream lift launch");
                break;
            }
            }
            if (rc) return rc;
            // (a packed Unwrap's prep reads no capacity: the placement writes the decode's into d.dc)
            const BatchArgs b{enc ? a.src : (const uint8_t*)sl.io.p, d.so, d.sl, enc ? (uint8_t*)sl.io.p : a.dst, d.dof,
                              a.kind == Stage::UNWRAP && placed ? nullptr : d.dc, d.out, m};
            // a packed stage places behind the previous stage's placement (lz4_packed.cuh); the next one follows
            const Placement pl = chained_placement(sl, d, async_fits(sl.meta.p, m), a.dst_total_cap, k > 0 ? &c->aslot[prev] : nullptr,
                                                   &carry->async[prev], &carry->async[s]);
            const int32_t hc_large = a.from == Source::CUT ? (a.op == Op::ENCODE_HC && a.block_size > 65536 ? m : 0)
                                                           : stage_hc_large(a.op, a.src_len, p.b0, p.b1);
            const int lanes = a.from == Source::LIFTED || a.from == Source::WALKED ? 0 : stage_lanes(c, a.op, a.src_len, a.dst_cap, p.b0, p.b1);
            rc = run_stage(c, a.kind, a.op, b, lanes, hc_large, packet_view(sl.meta.p, m), placed ? &pl : nullptr, framed ? d.aux : nullptr,
                           sl.stream);
            if (rc) return rc;
            // what lands, after its scan e: `bytes` dense bytes at `from` (dof, len), behind the previous stage's landing
            auto land = [&](cudaError_t e, const uint8_t* from, const int64_t* dof, const int32_t* len, int64_t bytes, int64_t* to_off,
                            int32_t* to_len) -> int {
                if (e == cudaSuccess && k > 0) e = cudaStreamWaitEvent(sl.stream, c->aslot[prev].carried, 0);
                if (e == cudaSuccess)
                    e = launch_land(from, dof, len, offs, m, bytes, k > 0 ? &carry->async[prev] : nullptr, a.dst_total_cap, a.dst, to_off,
                                    to_len, &carry->async[s], c->dev, sl.stream, &c->launches);
                if (e != cudaSuccess) return cuda_fail(e, "scan / landing launch");
                CU(cudaEventRecord(sl.carried, sl.stream));
                return LZ4B200_OK;
            };
            switch (a.kind) {
            case Stage::STREAM_ENCODE:      // the frames land, at their scan, of their sizes
                rc = land(write_frames(c, b, a.op == Op::ENCODE_HC, d.aux, offs, sl.scan.p, sl.scan.cap, (uint8_t*)sl.frames.p, sl.stream),
                          (const uint8_t*)sl.frames.p, offs, d.aux, p.sp.dsum + (int64_t)m * STREAM_HEADER_MAX, nullptr, nullptr);
                break;
            case Stage::FRAMED_DECODE:
                rc = launched(launch_stream_status(d.sl, d.aux, d.out, m, &carry->failed, sl.stream, &c->launches), "stream status launch");
                break;
            case Stage::CODEC:
            case Stage::WRAP_ENCODE:
                if (enc) {
                    rc = land(launch_compact(nullptr, nullptr, d.out, nullptr, offs, m, sl.scan.p, sl.scan.cap, c->dev, sl.stream, &c->launches),
                              (const uint8_t*)sl.io.p, d.dof, d.out, p.sp.dsum, a.out_off + p.b0, a.out_len + p.b0);
                    break;
                }
                [[fallthrough]];
            case Stage::PLACED_DECODE:
            case Stage::UNWRAP:
                if (a.from == Source::LIFTED)
                    rc = launched(launch_lift_status(a.src_cap, span, m, d.aux, d.out, sl.stream, &c->launches), "lift status launch");
                if (rc) return rc;
                CU(cudaMemcpyAsync(a.out_len + p.b0, d.out, sizeof(int32_t) * (size_t)m, cudaMemcpyDefault, sl.stream));
                if (placed) {
                    CU(cudaMemcpyAsync(a.out_off + p.b0, d.dof, sizeof(int64_t) * (size_t)m, cudaMemcpyDefault, sl.stream));
                    if (p.b1 == a.n) CU(cudaMemcpyAsync(a.out_off + a.n, &carry->async[s], sizeof(int64_t), cudaMemcpyDefault, sl.stream));
                }
                break;
            }
            if (rc) return rc;
        }
        return LZ4B200_OK;
    };
    // whatever was enqueued, the caller's stream joins it, and the chain and the metadata block are recorded behind it; an
    // LZ4Stream call whose stages are all in writes its size or status in between
    auto join = [&](bool all_in) -> int {
        for (int s = 0; s < used; s++) {
            CU(cudaEventRecord(c->aslot[s].done, c->aslot[s].stream));
            CU(cudaStreamWaitEvent(caller, c->aslot[s].done, 0));
        }
        const int last = (int)((plan.size() - 1) % NASYNC);
        int tail = LZ4B200_OK;
        if (all_in) switch (a.kind) {
        case Stage::STREAM_ENCODE:
            tail = launched(cudaMemcpyAsync(a.out_off, &carry->async[last], sizeof(int64_t), cudaMemcpyDefault, caller), "stream size copy");
            break;
        case Stage::FRAMED_DECODE:
            tail = launched(a.from == Source::WALKED ? launch_stream_walk_result(&carry->failed, carry->walk[last], a.out_off, caller, &c->launches)
                                                     : launch_stream_result(&carry->failed, a.total, a.out_off, caller, &c->launches),
                            "stream result launch");
            break;
        default: break;
        }
        CU(c->async_done.record(caller, Capture{}));
        if (blk) CU(cudaEventRecord(blk->done, caller));
        return tail;
    };
    int rc = stages();
    const int jr = join(rc == LZ4B200_OK);
    return rc ? rc : jr;
}

// The way into every asynchronous call, after its argument checks: the context's lock and device, the capture refusal,
// each pointer by the side it must be on (a packed call's out_off first, then out_off[0] = 0 if there is nothing to do;
// an LZ4Stream's headers are walked once src is known to be page-locked), then run_async.  The kernels reach the
// caller's memory at its device addresses; the copy engines take the caller's addresses as given.
int enter_async(lz4b200_ctx* c, AsyncCall a, void* stream, const char* what)
{
    CallGuard g(c); if (g.rc) return g.rc;
    int rc = refuse_capture(stream, what, false); if (rc) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    const bool lz4s = a.kind == Stage::STREAM_ENCODE || a.kind == Stage::FRAMED_DECODE, walked = a.from == Source::WALKED;
    const bool from_device = a.from == Source::DEVICE || a.from == Source::CUT;      // src device memory, dst page-locked
    void* at = nullptr;
    // p's device address, in `at`, and in p itself for a pointer the kernels take (use)
    auto reach = [&](auto*& p, bool device_ok, const char* name, bool use) {
        const int r = device_address(c, p, device_ok, name, &at);
        if (!r && use) p = static_cast<std::remove_reference_t<decltype(p)>>(at);
        return r;
    };
    if (a.out_off && !walked) {
        rc = reach(a.out_off, true, lz4s ? "out_size" : "out_off", a.from != Source::COPIED || lz4s); if (rc) return rc;
        if (lz4s ? a.stream_len == 0 : a.n == 0) { CU(cudaMemsetAsync(at, 0, sizeof(int64_t), st)); return LZ4B200_OK; }
    }
    if (a.n == 0 && !lz4s) return LZ4B200_OK;
    if (from_device) rc = check_side(c, a.src, true, "src");
    else if (a.src) rc = reach(a.src, false, "src", a.from != Source::COPIED);      // a walked call's src may be null
    if (!rc && a.from == Source::LIFTED) rc = reach(a.src_off, true, "src_off", false);
    if (!rc && walked) rc = reach(a.src_size, true, "src_size", true);
    if (rc) return rc;
    StreamEntries e;
    if (a.from == Source::COPIED && lz4s) {
        // src is final: a caller who knows the stream's length has its bytes in place
        a.total = stream_entries(a.src, a.stream_len, &e);
        if (a.total < 0) return fail((int)a.total, "malformed LZ4Stream");
        if (a.total > a.dst_total_cap || (a.total > 0 && !a.dst)) return fail(LZ4B200_E_ARG, "dst_cap < the decoded size");
        if (a.total == 0) { CU(cudaMemsetAsync(a.out_off, 0, sizeof(int64_t), st)); return LZ4B200_OK; }
        if (e.so.size() > (size_t)INT32_MAX) return fail(LZ4B200_E_ARG, "more than INT32_MAX non-empty chunks");
        a.n = (int32_t)e.so.size();
        a.src_off = e.so.data(); a.src_len = e.len.data(); a.dst_off = e.dof.data(); a.dst_cap = e.raw.data(); a.stored = e.stored.data();
    }
    if (from_device) rc = reach(a.dst, false, "dst", true);
    else if (a.dst) rc = check_side(c, a.dst, true, "dst");                            // a walked call's dst may be null
    if (!rc && a.out_len) rc = reach(a.out_len, true, "out_len", from_device);
    if (!rc && walked) rc = reach(a.out_off, true, "out_size", true);
    return rc ? rc : run_async(c, a, st);
}

// The capacities of n Wrap packets, src_len[i] + 8 (the largest a packet gets), into caps; an input whose packet would not
// fit an int32 is refused.  Packets that go into the caller's slots (slot_cap) must each fit their slot.
int wrap_caps(const int32_t* src_len, const int32_t* slot_cap, int32_t n, std::vector<int32_t>& caps)
{
    caps.resize((size_t)n);
    for (int32_t i = 0; i < n; i++) {
        if (src_len[i] < 0 || src_len[i] > INT32_MAX - WRAP_HEADER) return fail(LZ4B200_E_ARG, "input length: negative, or a packet above INT32_MAX bytes");
        if (slot_cap && (int64_t)slot_cap[i] < (int64_t)src_len[i] + WRAP_HEADER) return fail(LZ4B200_E_ARG, "dst_cap[i] < src_len[i] + 8");
        caps[i] = src_len[i] + WRAP_HEADER;
    }
    return LZ4B200_OK;
}

// The argument checks of the asynchronous packed encodes (the codec's blocks; Wrap packets, kind WRAP_ENCODE, whose
// capacities are their own), then enter_async.
int encode_async(lz4b200_ctx* c, Stage kind, int mode, const void* src, const int64_t* src_off, const int32_t* src_len,
                 const int32_t* dst_cap, void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n,
                 void* stream, const char* what)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (mode != LZ4B200_MODE_FAST && mode != LZ4B200_MODE_HC) return fail(LZ4B200_E_ARG, "unknown encoder mode");
    if (n < 0 || !out_off || dst_total_cap < 0) return fail(LZ4B200_E_ARG, "bad argument");
    const bool wrap = kind == Stage::WRAP_ENCODE;
    if (n > 0 && (!src || !src_off || !src_len || (!wrap && !dst_cap) || !dst || !out_len)) return fail(LZ4B200_E_ARG, "null argument");
    // a Wrap's dense slots hold whole packets
    std::vector<int32_t> pcap;
    int rc = wrap ? wrap_caps(src_len, nullptr, n, pcap) : check_lengths(src_len, dst_cap, n, "block"); if (rc) return rc;
    return enter_async(c, {kind, encode_op(mode == LZ4B200_MODE_HC), Source::DEVICE, (const uint8_t*)src, src_off, src_len, (uint8_t*)dst,
                           nullptr, wrap ? pcap.data() : dst_cap, out_len, n, out_off, dst_total_cap}, stream, what);
}

// The argument checks of the asynchronous decodes (the codec's blocks; Unwrap packets, kind UNWRAP) into the caller's
// slots or packed (out_off, dst_total_cap; no dst_off, dst_cap), then enter_async.
int decode_async(lz4b200_ctx* c, Stage kind, Op op, bool packed, const void* src, const int64_t* src_off, const int32_t* src_len,
                 void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, int64_t* out_off,
                 int64_t dst_total_cap, void* stream, const char* what)
{
    const char* unit = kind == Stage::UNWRAP ? "packet" : "block";
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (packed && (n < 0 || !out_off || dst_total_cap < 0)) return fail(LZ4B200_E_ARG, "bad argument");
    if (n < 0) return fail(LZ4B200_E_ARG, std::string("negative ") + unit + " count");
    if (n > 0 && (!src || !src_off || !src_len || !dst || (!packed && (!dst_off || !dst_cap)) || !out_len))
        return fail(LZ4B200_E_ARG, "null argument");
    int rc = check_lengths(src_len, dst_cap, n, unit); if (rc) return rc;
    return enter_async(c, {kind, op, Source::COPIED, (const uint8_t*)src, src_off, src_len, (uint8_t*)dst, dst_off, dst_cap, out_len, n,
                           out_off, dst_total_cap}, stream, what);
}

// The argument checks of the decode and Unwrap whose offsets src_off (n + 1) are read on the device, and each block's
// bound (compress_bound(dst_cap[i]), or an Unwrap packet's dst_cap[i] + 8, at most INT32_MAX); then enter_async.
int decode_at_async(lz4b200_ctx* c, Stage kind, Op op, const void* src, int64_t src_cap, const int64_t* src_off, void* dst,
                 const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream, const char* what)
{
    const bool unwrap = kind == Stage::UNWRAP;
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0 || src_cap < 0) return fail(LZ4B200_E_ARG, "bad argument");
    if (n > 0 && (!src || !src_off || !dst || !dst_off || !dst_cap || !out_len)) return fail(LZ4B200_E_ARG, "null argument");
    AsyncCall a{kind, op, Source::LIFTED, (const uint8_t*)src, src_off, nullptr, (uint8_t*)dst, dst_off, dst_cap, out_len, n, nullptr, 0,
                src_cap};
    a.bound.resize((size_t)n);
    for (int32_t i = 0; i < n; i++) {
        if (dst_cap[i] < 0) return fail(LZ4B200_E_ARG, std::string("negative ") + (unwrap ? "packet" : "block") + " capacity");
        a.bound[i] = unwrap ? (int32_t)std::min<int64_t>((int64_t)dst_cap[i] + WRAP_HEADER, INT32_MAX)
                            : (int32_t)std::min<int64_t>((int64_t)dst_cap[i] + dst_cap[i] / 255 + 16, INT32_MAX);
    }
    return enter_async(c, std::move(a), stream, what);
}

// The argument checks of the LZ4Stream decode whose size S (*src_size) the device wrote, then enter_async.  src may be
// null when src_cap == 0, dst when dst_cap == 0.
int walked_async(lz4b200_ctx* c, const void* src, int64_t src_cap, const int64_t* src_size, int32_t block_size, void* dst,
                 int64_t dst_cap, int64_t* out_size, void* stream, const char* what)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (src_cap < 0 || dst_cap < 0) return fail(LZ4B200_E_ARG, "bad argument");
    if (block_size < 1 || block_size > INT32_MAX - STREAM_HEADER_MAX) return fail(LZ4B200_E_ARG, "block_size: a chunk's frame must fit an int32");
    if (!src_size || !out_size || (src_cap > 0 && !src) || (dst_cap > 0 && !dst)) return fail(LZ4B200_E_ARG, "null argument");
    return enter_async(c, {Stage::FRAMED_DECODE, Op::DECODE_KNOWN, Source::WALKED, (const uint8_t*)src, nullptr, nullptr, (uint8_t*)dst,
                           nullptr, nullptr, nullptr, 0, out_size, dst_cap, src_cap, src_size, 0, block_size}, stream, what);
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
    if (mem == LZ4B200_MEM_DEVICE) {
        DeviceCall call(c, stream); if (call.rc) return call.rc;
        int rc = call.enter(need_of(c, n, op == Op::ENCODE_HC ? HC : 0, measure ? 0 : 1)); if (rc) return rc;
        BatchArgs a{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, dst_off, dst_cap, out_len, n};
        return run_device(c, a, op, call.st, 0, -1, call.cap);
    }
    CallGuard g(c); if (g.rc) return g.rc;
    const bool src_dev = mem == LZ4B200_MEM_DEVICE_TO_HOST, dst_dev = mem == LZ4B200_MEM_HOST_TO_DEVICE;
    if (mem != LZ4B200_MEM_HOST && !src_dev && !dst_dev)
        return fail(LZ4B200_E_ARG, "mem must be LZ4B200_MEM_HOST, _DEVICE, _DEVICE_TO_HOST or _HOST_TO_DEVICE");
    if (src_dev || dst_dev) {
        int rc = refuse_capture(stream, "a mixed-memory batch"); if (rc) return rc;
        // the measure pass has no destination: MEM_HOST and MEM_DEVICE already cover both places its source can be
        if (measure) return fail(LZ4B200_E_ARG, "measure_batch takes LZ4B200_MEM_HOST or LZ4B200_MEM_DEVICE");
        rc = check_side(c, src, src_dev, "src"); if (rc) return rc;
        rc = check_side(c, dst, dst_dev, "dst"); if (rc) return rc;
    }
    return run_host(c, Stage::CODEC, op, (const uint8_t*)src, src_off, src_len, (uint8_t*)dst, dst_off, dst_cap, out_len, n, out_off,
                    dst_total_cap, src_dev, dst_dev, (cudaStream_t)stream);
}

// The packed encode into host memory, from host memory (MEM_HOST) or device memory (MEM_DEVICE_TO_HOST): n == 0 writes
// out_off[0] = 0.
int encode_packed(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, const int32_t* dst_cap, void* dst,
                  int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n, int mode, int mem, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (mode != LZ4B200_MODE_FAST && mode != LZ4B200_MODE_HC) return fail(LZ4B200_E_ARG, "unknown encoder mode");
    if (n < 0 || !out_off) return fail(LZ4B200_E_ARG, "bad argument");
    if (n == 0) { out_off[0] = 0; return LZ4B200_OK; }
    return batch(c, src, src_off, src_len, dst, nullptr, dst_cap, out_len, n, encode_op(mode == LZ4B200_MODE_HC), mem, stream, out_off,
                 dst_total_cap);
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

// The arguments of an LZ4Stream encode of n bytes in block_size chunks into dst_cap bytes, synchronous or not.
int stream_encode_args(const lz4b200_ctx* c, const void* src, int64_t n, int32_t block_size, const void* dst, int64_t dst_cap)
{
    if (!c || n < 0 || block_size < 1 || (n > 0 && (!src || !dst))) return fail(LZ4B200_E_ARG, "bad argument");
    if (std::min<int64_t>(block_size, n) > INT32_MAX - STREAM_HEADER_MAX) return fail(LZ4B200_E_ARG, "a chunk's frame must fit an int32");
    if (dst_cap < lz4b200_stream_bound(n, block_size)) return fail(LZ4B200_E_ARG, "dst_cap < lz4b200_stream_bound(n, block_size)");
    return LZ4B200_OK;
}

// The LZ4Stream of n bytes in host or device memory (src_dev), written into host memory: each run of chunks is encoded
// (capacity = the chunk's length, LZ4Stream.cs:243-246) and its frames land back to back (STREAM_ENCODE, APPEND).  Returns
// the stream's size.  Only a chunk whose frame does not fit an int32 is refused for its size.
int64_t stream_encode(lz4b200_ctx* c, const void* src, int64_t n, int32_t block_size, int high_compression, void* dst,
                      int64_t dst_cap, bool src_dev, void* stream)
{
    if (int rc = stream_encode_args(c, src, n, block_size, dst, dst_cap)) return rc;
    if (n == 0) return 0;
    CallGuard g(c); if (g.rc) return g.rc;
    if (src_dev) {
        int rc = refuse_capture(stream, "lz4b200_stream_encode_from_device"); if (rc) return rc;
        rc = check_side(c, src, true, "src"); if (rc) return rc;
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
    if (dst_dev) {
        int rc = refuse_capture(stream, "lz4b200_stream_decode_to_device"); if (rc) return rc;
        rc = check_side(c, src, false, "src"); if (rc) return rc;
    }
    StreamEntries e;
    const int64_t total = stream_entries((const uint8_t*)src, n, &e);
    if (total < 0) return fail((int)total, "malformed LZ4Stream");
    if (total > dst_cap || (total > 0 && !dst)) return fail(LZ4B200_E_ARG, "dst_cap < the decoded size");
    if (total == 0) return 0;
    if (dst_dev) { int rc = check_side(c, dst, true, "dst"); if (rc) return rc; }
    std::vector<int32_t> res;
    const int64_t entries = (int64_t)e.so.size();
    for (int64_t e0 = 0; e0 < entries; e0 += STREAM_RUN_CHUNKS) {
        const int32_t m = (int32_t)std::min(STREAM_RUN_CHUNKS, entries - e0);
        res.assign(m, -1);
        int rc = run_host(c, Stage::FRAMED_DECODE, Op::DECODE_KNOWN, (const uint8_t*)src, e.so.data() + e0, e.len.data() + e0,
                          (uint8_t*)dst, e.dof.data() + e0, e.raw.data() + e0, res.data(), m, nullptr, 0, false, dst_dev,
                          (cudaStream_t)stream, e.stored.data() + e0);
        if (rc) return rc;
        // a compressed chunk decodes from exactly its compLen bytes (LZ4Codec.Safe.cs:539-542)
        for (int32_t i = 0; i < m; i++)
            if (!e.stored[e0 + i] && res[i] != e.len[e0 + i]) return fail(LZ4B200_E_FORMAT, "a chunk does not decode to its compressed length");
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
    std::vector<int32_t> pcap;
    int rc = wrap_caps(src_len, dst_off ? dst_cap : nullptr, n, pcap); if (rc) return rc;
    CallGuard g(c); if (g.rc) return g.rc;
    if (src_dev) {
        rc = refuse_capture(stream, "a Wrap from device memory"); if (rc) return rc;
        rc = check_side(c, src, true, "src"); if (rc) return rc;
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
        int rc = refuse_capture(stream, "an Unwrap into device memory"); if (rc) return rc;
        rc = check_side(c, src, false, "src"); if (rc) return rc;
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
    cudaError_t e = cudaMalloc(&c->counters, sizeof(uint32_t) * (NCOUNTER + 4 * NCAPTURED));
    if (e == cudaSuccess) e = cudaMalloc(&c->carry, sizeof(Carry));
    for (Chain* ch : {&c->hc_done, &c->compact_done, &c->async_done}) {
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ch->done, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ch->inner, cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->entry, cudaEventDisableTiming);
    for (Slot& s : c->slot) if (e == cudaSuccess) e = create_slot(s);
    for (AsyncSlot& s : c->aslot) if (e == cudaSuccess) e = create_slot(s);
    if (e != cudaSuccess) { int rc = cuda_fail(e, "context creation"); lz4b200_destroy(c); return rc; }
    *out = c;
    return LZ4B200_OK;
}

void lz4b200_destroy(lz4b200_ctx* c)
{
    if (!c) return;
    DeviceGuard g(c->device);
    cudaDeviceSynchronize();
    for (Slot& s : c->slot) destroy_slot(s);
    for (AsyncSlot& s : c->aslot) destroy_slot(s);
    for (auto& b : c->meta_pool) if (b->done) cudaEventDestroy(b->done);
    for (Chain* ch : {&c->hc_done, &c->compact_done, &c->async_done}) {
        if (ch->done) cudaEventDestroy(ch->done);
        if (ch->inner) cudaEventDestroy(ch->inner);
    }
    if (c->entry) cudaEventDestroy(c->entry);
    if (c->counters) cudaFree(c->counters);
    if (c->carry) cudaFree(c->carry);
    for (void* p : c->retired) cudaFree(p);
    delete c;                                      // (the buffers free themselves, on the context's device)
}

int lz4b200_synchronize(lz4b200_ctx* c)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    DeviceGuard g(c->device);
    for (int i = 0; i < NSLOT; i++) CU(cudaStreamSynchronize(c->slot[i].stream));
    for (int i = 0; i < NASYNC; i++) CU(cudaStreamSynchronize(c->aslot[i].stream));
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
    return encode_packed(c, src, src_off, src_len, dst_cap, dst, dst_total_cap, out_off, out_len, n, mode, LZ4B200_MEM_HOST, nullptr);
}

int lz4b200_encode_batch_packed_from_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                            const int32_t* dst_cap, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                            int32_t* out_len, int32_t n, int mode, void* stream)
{
    return encode_packed(c, src, src_off, src_len, dst_cap, dst, dst_total_cap, out_off, out_len, n, mode, LZ4B200_MEM_DEVICE_TO_HOST,
                         stream);
}

// ---- between device memory and page-locked host memory without blocking: run_async -----------------------------------
int lz4b200_encode_batch_packed_from_device_async(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                                  const int32_t* dst_cap, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                                  int32_t* out_len, int32_t n, int mode, void* stream)
{
    return encode_async(c, Stage::CODEC, mode, src, src_off, src_len, dst_cap, dst, dst_total_cap, out_off, out_len, n, stream,
                        "lz4b200_encode_batch_packed_from_device_async");
}

int lz4b200_decode_batch_to_device_async(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                         const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, int known_len,
                                         void* stream)
{
    return decode_async(c, Stage::CODEC, known_len ? Op::DECODE_KNOWN : Op::DECODE_UNKNOWN, false, src, src_off, src_len, dst, dst_off,
                        dst_cap, out_len, n, nullptr, 0, stream, "lz4b200_decode_batch_to_device_async");
}

int lz4b200_decode_batch_packed_to_device_async(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                                void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n,
                                                void* stream)
{
    return decode_async(c, Stage::PLACED_DECODE, Op::DECODE_UNKNOWN, true, src, src_off, src_len, dst, nullptr, nullptr, out_len, n,
                        out_off, dst_total_cap, stream, "lz4b200_decode_batch_packed_to_device_async");
}

int lz4b200_wrap_batch_packed_from_device_async(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                                int high_compression, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                                int32_t* out_len, int32_t n, void* stream)
{
    return encode_async(c, Stage::WRAP_ENCODE, high_compression ? LZ4B200_MODE_HC : LZ4B200_MODE_FAST, src, src_off, src_len, nullptr,
                        dst, dst_total_cap, out_off, out_len, n, stream, "lz4b200_wrap_batch_packed_from_device_async");
}

int lz4b200_unwrap_batch_to_device_async(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                         const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream)
{
    return decode_async(c, Stage::UNWRAP, Op::DECODE_KNOWN, false, src, src_off, src_len, dst, dst_off, dst_cap, out_len, n, nullptr, 0,
                        stream, "lz4b200_unwrap_batch_to_device_async");
}

int lz4b200_unwrap_batch_packed_to_device_async(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                                void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n,
                                                void* stream)
{
    return decode_async(c, Stage::UNWRAP, Op::DECODE_KNOWN, true, src, src_off, src_len, dst, nullptr, nullptr, out_len, n, out_off,
                        dst_total_cap, stream, "lz4b200_unwrap_batch_packed_to_device_async");
}

// The decode and the Unwrap whose offsets the device wrote (an asynchronous packed encode's or Wrap's out_off), staged by
// the lift kernel (lz4_lift.cuh).
int lz4b200_decode_batch_to_device_at_async(lz4b200_ctx* c, const void* src, int64_t src_cap, const int64_t* src_off, void* dst,
                                            const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, int known_len,
                                            void* stream)
{
    return decode_at_async(c, Stage::CODEC, known_len ? Op::DECODE_KNOWN : Op::DECODE_UNKNOWN, src, src_cap, src_off, dst, dst_off, dst_cap,
                        out_len, n, stream, "lz4b200_decode_batch_to_device_at_async");
}

int lz4b200_unwrap_batch_to_device_at_async(lz4b200_ctx* c, const void* src, int64_t src_cap, const int64_t* src_off, void* dst,
                                            const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream)
{
    return decode_at_async(c, Stage::UNWRAP, Op::DECODE_KNOWN, src, src_cap, src_off, dst, dst_off, dst_cap, out_len, n, stream,
                        "lz4b200_unwrap_batch_to_device_at_async");
}

// An LZ4Stream without blocking: the encode's chunk table is computed on the device and its frames land like the packed
// encode's blocks (STREAM_ENCODE); the decode's headers are walked on the host during the call (FRAMED_DECODE).
int lz4b200_stream_encode_from_device_async(lz4b200_ctx* c, const void* src, int64_t n, int32_t block_size, int high_compression,
                                            void* dst, int64_t dst_cap, int64_t* out_size, void* stream)
{
    if (block_size > INT32_MAX - STREAM_HEADER_MAX) return fail(LZ4B200_E_ARG, "block_size: a chunk's frame must fit an int32");
    if (int rc = stream_encode_args(c, src, n, block_size, dst, dst_cap)) return rc;
    if (!out_size) return fail(LZ4B200_E_ARG, "bad argument");
    return enter_async(c, {Stage::STREAM_ENCODE, encode_op(high_compression != 0), Source::CUT, (const uint8_t*)src, nullptr, nullptr,
                           (uint8_t*)dst, nullptr, nullptr, nullptr, 0, out_size, dst_cap, 0, nullptr, n, block_size},
                       stream, "lz4b200_stream_encode_from_device_async");
}

int lz4b200_stream_decode_to_device_async(lz4b200_ctx* c, const void* src, int64_t n, void* dst, int64_t dst_cap, int64_t* out_size,
                                          void* stream)
{
    if (!c || n < 0 || (n > 0 && !src) || !out_size) return fail(LZ4B200_E_ARG, "bad argument");
    return enter_async(c, {Stage::FRAMED_DECODE, Op::DECODE_KNOWN, Source::COPIED, (const uint8_t*)src, nullptr, nullptr, (uint8_t*)dst,
                           nullptr, nullptr, nullptr, 0, out_size, dst_cap, 0, nullptr, n}, stream, "lz4b200_stream_decode_to_device_async");
}

// The LZ4Stream decode whose size an asynchronous encode wrote on the device: its headers are walked there (walked_async).
int lz4b200_stream_decode_to_device_at_async(lz4b200_ctx* c, const void* src, int64_t src_cap, const int64_t* src_size,
                                             int32_t block_size, void* dst, int64_t dst_cap, int64_t* out_size, void* stream)
{
    return walked_async(c, src, src_cap, src_size, block_size, dst, dst_cap, out_size, stream, "lz4b200_stream_decode_to_device_at_async");
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

// run_placed_decode, all enqueued on `stream`, placed in one piece by the call scratch.
int lz4b200_decode_batch_packed(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len,
                                void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0 || !out_off || dst_total_cap < 0) return fail(LZ4B200_E_ARG, "bad argument");
    DeviceCall call(c, stream); if (call.rc) return call.rc;
    if (n == 0) { CU(cudaMemsetAsync(out_off, 0, sizeof(int64_t), call.st)); return LZ4B200_OK; }     // out_off[0] = total = 0
    if (!src || !src_off || !src_len || !dst || !out_len) return fail(LZ4B200_E_ARG, "null argument");
    int rc = call.enter(need_of(c, n, SCAN | CAPS, 1)); if (rc) return rc;
    int32_t* caps = (int32_t*)c->packed_caps.p;
    const Placement pl{out_off, c->compact_tmp.p, c->compact_tmp.cap, dst_total_cap, 0, caps, (int*)(caps + n)};
    const BatchArgs a{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, out_off, caps, out_len, n};
    rc = run_placed_decode(c, a, pl, call.st, call.cap); if (rc) return rc;
    return call.done();
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
    int rc = refuse_capture(stream, "lz4b200_decode_batch_packed_to_device"); if (rc) return rc;
    rc = check_side(c, src, false, "src"); if (rc) return rc;
    rc = check_side(c, dst, true, "dst"); if (rc) return rc;
    return run_host(c, Stage::PLACED_DECODE, Op::DECODE_UNKNOWN, (const uint8_t*)src, src_off, src_len, (uint8_t*)dst, nullptr,
                    nullptr, out_len, n, out_off, dst_total_cap, false, true, (cudaStream_t)stream);
}

int lz4b200_compact(lz4b200_ctx* c, const void* slots, const int64_t* slot_off, const int32_t* len, void* packed,
                    int64_t* out_off, int32_t n, void* stream)
{
    if (!c || !slot_off || !len || !out_off || n < 0) return fail(LZ4B200_E_ARG, "bad argument");
    DeviceCall call(c, stream); if (call.rc) return call.rc;
    if (n == 0) { CU(cudaMemsetAsync(out_off, 0, sizeof(int64_t), call.st)); return LZ4B200_OK; }     // out_off[0] = total = 0
    int rc = call.enter(need_of(c, n, SCAN, 0)); if (rc) return rc;
    cudaError_t e = launch_compact((const uint8_t*)slots, slot_off, len, (uint8_t*)packed, out_off, n,
                                   c->compact_tmp.p, c->compact_tmp.cap, c->dev, call.st, &c->launches);
    if (e != cudaSuccess) return cuda_fail(e, "compact launch");
    return call.done();
}

// ---- Wrap / Unwrap packets in device memory (lz4_wrap.cuh): prep -> the batch codec, unchanged -> finish, on `stream` ----
int lz4b200_wrap_batch_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, int high_compression,
                              void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0) return fail(LZ4B200_E_ARG, "negative packet count");
    DeviceCall call(c, stream); if (call.rc) return call.rc;
    if (n == 0) return LZ4B200_OK;
    if (!src || !src_off || !src_len || !dst || !dst_off || !dst_cap || !out_len) return fail(LZ4B200_E_ARG, "null argument");
    int rc = call.enter(need_of(c, n, WRAP | (high_compression ? HC : 0), 1)); if (rc) return rc;
    // the same encode as lz4b200_encode_batch(MEM_DEVICE): HC sizes its arena as if every block were above 64 KiB
    const BatchArgs a{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, dst_off, dst_cap, out_len, n};
    rc = run_wrap(c, a, wrap_scratch_at(c->wrap_tmp.p, n), encode_op(high_compression != 0), call.st, -1, call.cap); if (rc) return rc;
    return call.done();
}

int lz4b200_unwrap_batch_device(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0) return fail(LZ4B200_E_ARG, "negative packet count");
    DeviceCall call(c, stream); if (call.rc) return call.rc;
    if (n == 0) return LZ4B200_OK;
    if (!src || !src_off || !src_len || !dst || !dst_off || !dst_cap || !out_len) return fail(LZ4B200_E_ARG, "null argument");
    int rc = call.enter(need_of(c, n, WRAP, 1)); if (rc) return rc;
    const BatchArgs a{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, dst_off, dst_cap, out_len, n};
    rc = run_unwrap(c, a, wrap_scratch_at(c->wrap_tmp.p, n), call.st, call.cap); if (rc) return rc;
    return call.done();
}

// sizes from the headers -> scan into out_off -> capacities + "fits" -> decode and stored copies, both behind the flag
int lz4b200_unwrap_batch_packed(lz4b200_ctx* c, const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n, void* stream)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (n < 0) return fail(LZ4B200_E_ARG, "negative packet count");
    DeviceCall call(c, stream); if (call.rc) return call.rc;
    if (!out_off || dst_total_cap < 0) return fail(LZ4B200_E_ARG, "bad argument");
    if (n == 0) { CU(cudaMemsetAsync(out_off, 0, sizeof(int64_t), call.st)); return LZ4B200_OK; }     // out_off[0] = total = 0
    if (!src || !src_off || !src_len || !dst || !out_len) return fail(LZ4B200_E_ARG, "null argument");
    int rc = call.enter(need_of(c, n, SCAN | CAPS | WRAP, 1)); if (rc) return rc;
    int32_t* caps = (int32_t*)c->packed_caps.p;
    const Placement pl{out_off, c->compact_tmp.p, c->compact_tmp.cap, dst_total_cap, 0, caps, (int*)(caps + n)};
    const BatchArgs a{(const uint8_t*)src, src_off, src_len, (uint8_t*)dst, out_off, nullptr, out_len, n};
    rc = run_unwrap(c, a, wrap_scratch_at(c->wrap_tmp.p, n), call.st, call.cap, &pl); if (rc) return rc;
    return call.done();
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

// Everything a device call of at most max_blocks blocks takes from the shared scratch, grown as an eager call grows it.
int lz4b200_reserve(lz4b200_ctx* c, int32_t max_blocks, int high_compression)
{
    if (!c) return fail(LZ4B200_E_ARG, "null context");
    if (max_blocks < 0) return fail(LZ4B200_E_ARG, "negative block count");
    if (max_blocks == 0) return LZ4B200_OK;
    CallGuard g(c); if (g.rc) return g.rc;
    return grow_scratch(c, need_of(c, max_blocks, SCAN | CAPS | WRAP | (high_compression ? HC : 0), 0));
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
        c->hc_arena.drop(c->retired);
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
