/*
 * lz4b200.h -- C ABI of liblz4b200.so: the H100 (sm_90a) LZ4 r93 block codec behind lz4net's service boundary.
 *
 * This is the drop-in boundary of the path (SURVEY.md 8b).  lz4net's native services (LZ4mm / LZ4cc) reach the
 * codec through exactly four C functions (src/LZ4cc/LZ4Codec.64.cpp:35,88,95,143 -> original/lz4.h:59-60,101,116,
 * original/lz4hc.h:57); a `CudaLZ4Service : ILZ4Service` (src/LZ4/ILZ4Service.cs:30-36) binds the entry points
 * below with [DllImport] exactly like CppMM64LZ4Service (src/LZ4/Services/CppMM64LZ4Service.cs:38-51) binds those.
 * INTEGRATION.md shows the managed stub.  Plain pointers and sizes only; no torch / CUDA types in any signature
 * (a `void* stream` is a cudaStream_t passed opaquely; NULL = the CUDA default stream, as everywhere in CUDA).
 *
 * Conventions shared with the reference:
 *   - encoders return bytes written, 0 = output too small / failed              (original/lz4.h:48-60)
 *   - known-size decode returns bytes READ from the source, < 0 = malformed     (original/lz4.h:96-101)
 *   - unknown-size decode returns bytes WRITTEN, < 0 = malformed                (original/lz4.h:104-116)
 *   - compressed bytes are identical to lz4net's LZ4Codec.Encode / EncodeHC on the same input
 * There is no CPU fallback: every entry point fails (LZ4B200_E_*) when no sm_90 device / kernel image is usable.
 */
#ifndef LZ4B200_H
#define LZ4B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LZ4B200_VERSION 100            /* 0.1.0 */

/* encoder selection (ILZ4Service.Encode vs EncodeHC, src/LZ4/ILZ4Service.cs:33-34) */
#define LZ4B200_MODE_FAST 0
#define LZ4B200_MODE_HC   1

/* where the buffers of a batch call live */
#define LZ4B200_MEM_HOST   0           /* src/dst/offset/length arrays are host memory; copies are inside the call */
#define LZ4B200_MEM_DEVICE 1           /* everything is device memory on the context's GPU; the call only enqueues */
/* Mixed memory (encode_batch / decode_batch; not measure_batch, which has no destination).  The offset, length and out_len
 * arrays are host memory.  Only compressed bytes cross PCIe, in one direction; device scratch stays at the host pipeline's
 * per-stage size whatever the batch.  Contract of every mixed call:
 *   - synchronous, like MEM_HOST;
 *   - its device reads and writes are ordered after all work enqueued on `stream` before the call (a kernel that fills
 *     src, or one still reading the old contents of dst), and every device access is complete when it returns;
 *   - out_len[i] and the bytes block i produced equal what MEM_DEVICE and MEM_HOST give for the same block;
 *   - a host destination receives only the bytes each block produced, as with MEM_HOST; a device destination is written
 *     only inside [dst_off[i], dst_off[i] + dst_cap[i]), as with MEM_DEVICE;
 *   - LZ4B200_E_ARG when the device side is not memory of the context's GPU, or the host side is device memory. */
#define LZ4B200_MEM_DEVICE_TO_HOST 2   /* src: device memory of the context's GPU; dst: host memory, pageable or page-locked */
#define LZ4B200_MEM_HOST_TO_DEVICE 3   /* src: host memory; dst: device memory of the context's GPU */

/* status codes (batch / context calls).  Per-block results are reported in out_len[], never here. */
#define LZ4B200_OK            0
#define LZ4B200_E_ARG        -1
#define LZ4B200_E_NODEVICE   -2        /* no CUDA device, or not compute capability 9.x */
#define LZ4B200_E_CUDA       -3        /* a CUDA runtime call failed; see lz4b200_last_error() */
#define LZ4B200_E_NOMEM      -4
#define LZ4B200_E_FORMAT     -5        /* malformed LZ4Stream / Wrap framing, or a chunk that does not decode */

typedef struct lz4b200_ctx lz4b200_ctx;

int         lz4b200_version(void);
const char* lz4b200_last_error(void);                 /* thread-local, never NULL */
int         lz4b200_device_count(void);               /* usable (cc 9.x) devices; 0 if none */

/* A context owns one device's stream, scratch (HC chain tables, staging) and tuning knobs.  Unlike the reference
 * (stateless: tables are allocated per call, src/LZ4ps/LZ4Codec.Safe.cs:407) the GPU path has state.
 * Contexts are internally locked: one batch call at a time per context; use one context per caller thread/GPU. */
int  lz4b200_create(lz4b200_ctx** out, int device);
void lz4b200_destroy(lz4b200_ctx* ctx);
int  lz4b200_synchronize(lz4b200_ctx* ctx);           /* wait for everything enqueued through this context */

/* LZ4_compressBound (original/lz4.h:85) == LZ4Codec.MaximumOutputLength (src/LZ4/LZ4Codec.cs:313-316) */
int  lz4b200_compress_bound(int input_size);

/* ---- batched entry points: n_blocks independent blocks, one launch -------------------------------------------
 * Block i reads  src + src_off[i], src_len[i] bytes   and writes at  dst + dst_off[i], at most dst_cap[i] bytes.
 * out_len[i] receives the per-block return value of the corresponding single-block function below.
 *
 * encode:  LZ4_compress_limitedOutput / LZ4_compressHC_limitedOutput semantics per block (0 = did not fit).
 * decode:  known_len != 0 -> LZ4_uncompress (dst_cap[i] is the exact decoded size; out_len[i] = bytes read,
 *                            the caller compares it with src_len[i] like src/LZ4cc/LZ4Codec.64.cpp:88-93);
 *          known_len == 0 -> LZ4_uncompress_unknownOutputSize (dst_cap[i] = capacity; out_len[i] = bytes written).
 * MEM_DEVICE: asynchronous on `stream`; MEM_HOST: synchronous, chunked + overlapped copies inside the call;
 * MEM_DEVICE_TO_HOST / MEM_HOST_TO_DEVICE: synchronous like MEM_HOST, ordered behind `stream` (see above).
 * Returns LZ4B200_OK or a negative status; malformed / too-small blocks are NOT a call failure. */
int lz4b200_encode_batch(lz4b200_ctx* ctx,
                         const void* src, const int64_t* src_off, const int32_t* src_len,
                         void* dst, const int64_t* dst_off, const int32_t* dst_cap,
                         int32_t* out_len, int32_t n_blocks, int mode, int mem, void* stream);

int lz4b200_decode_batch(lz4b200_ctx* ctx,
                         const void* src, const int64_t* src_off, const int32_t* src_len,
                         void* dst, const int64_t* dst_off, const int32_t* dst_cap,
                         int32_t* out_len, int32_t n_blocks, int known_len, int mem, void* stream);

/* ---- decoded sizes without decoding, and a decode whose output the library sizes itself ---------------------------
 * Raw LZ4 blocks do not store their decoded size (lz4net's LZ4Codec.Decode(..., knownOutputLength: false) leaves the
 * capacity to the caller).  The decoders' accept / reject decisions depend on the stream's structure alone, so a pass
 * over the headers that skips the payload predicts their result exactly, and validates a batch before any output
 * buffer is committed.
 *
 * measure_batch: out_len[i] = what lz4b200_decode_batch (same arguments) would store; nothing is decoded or written.
 *   Non-negative values are equal, negative ones agree in sign.  dst_cap may be NULL when known_len == 0 (capacity
 *   INT32_MAX per block; LZ4B200_E_ARG otherwise).  MEM_DEVICE: asynchronous on `stream`; MEM_HOST: synchronous; the
 *   mixed values are LZ4B200_E_ARG. */
int lz4b200_measure_batch(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                          const int32_t* dst_cap, int32_t* out_len, int32_t n_blocks, int known_len, int mem, void* stream);

/* decode_batch_packed (device memory only, asynchronous on `stream`, no host synchronisation): unknown-size decode into
 * PACKED output.  Every block is measured (capacity INT32_MAX); out_off[0..n] (int64, n_blocks+1 entries) = exclusive
 * prefix sum of max(size, 0), out_off[n] the total.  If out_off[n] <= dst_total_cap, block i is decoded to
 * dst + out_off[i] with capacity = its measured size and out_len[i] is the decoder's result (a malformed block reports a
 * negative value and occupies no bytes).  Otherwise dst is not touched and out_len[i] holds the measured sizes: allocate
 * out_off[n] bytes and call again.
 * Blocks in host memory wanted in device memory: lz4b200_decode_batch_packed_to_device below.  There is no form with a
 * host DESTINATION: the host pipeline sizes the device output buffer of a chunk by decoded bytes, which this call learns
 * only on the device.  Callers who want the output in host memory use lz4b200_measure_batch, then lz4b200_decode_batch. */
int lz4b200_decode_batch_packed(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n_blocks,
                                void* stream);

/* decode_batch_packed_to_device: the same for blocks in host memory (a file, a key-value store, a socket: compressed
 * lengths only) wanted decoded in device memory.  src: host memory, pageable or page-locked; dst: device memory of the
 * context's GPU; src_off, src_len, out_off (n_blocks+1 entries) and out_len are host arrays.  The contract of every mixed
 * call (LZ4B200_MEM_HOST_TO_DEVICE above): synchronous, ordered behind the work already queued on `stream`, LZ4B200_E_ARG
 * when src is device memory or dst is not memory of the context's GPU; only the compressed bytes cross PCIe, ONCE (not
 * once to be measured and once to be decoded), and device scratch stays at the per-stage size whatever n_blocks is.
 *   - out_off[0..n] = exclusive prefix sum of max(size_i, 0), size_i = what lz4b200_measure_batch(known_len = 0, dst_cap =
 *     NULL) reports for block i; out_off[n] = the total.  They are filled whether the total fits or not.
 *   - out_off[n] <= dst_total_cap: block i is decoded to dst + out_off[i] with capacity size_i; out_off, out_len and the
 *     bytes dst[0, out_off[n]) equal what lz4b200_decode_batch_packed gives for a device copy of the batch.  A malformed
 *     block reports a negative out_len[i] and occupies no bytes: that block's status, not the call's.
 *   - out_off[n] > dst_total_cap: still LZ4B200_OK.  Nothing outside [dst, dst + dst_total_cap) is written, the bytes
 *     inside it are unspecified, and out_len[i] is non-negative exactly for the well-formed blocks, where it equals size_i.
 *     Allocate out_off[n] bytes and call again.  This is weaker than lz4b200_decode_batch_packed's "dst is not touched", on
 *     purpose: the batch is decoded a pipeline stage at a time, the total is known only when the last stage has been
 *     uploaded, and holding the decoded output back until then would take the second pass over the compressed bytes that
 *     this call exists to avoid.  (A stage is decoded when everything up to its end fits.)
 *   - n_blocks == 0 is LZ4B200_OK with out_off[0] = 0; a negative src_len[i] is LZ4B200_E_ARG before any device work. */
int lz4b200_decode_batch_packed_to_device(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                          void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len,
                                          int32_t n_blocks, void* stream);

/* Host-memory encode with PACKED output: block i's compressed bytes land at dst + out_off[i] (out_off has n_blocks+1
 * entries; out_off[n_blocks] = total bytes written <= dst_total_cap), back to back in block order -- the layout the
 * LZ4Stream chunk writer (src/LZ4/LZ4Stream.cs:262-266) and any transport want, and the one that moves only compLen
 * bytes per block back over PCIe.  dst_cap[i] is still the per-block limit of LZ4_compress_limitedOutput (a block that
 * does not fit reports out_len[i] = 0 and occupies no bytes). */
int lz4b200_encode_batch_packed(lz4b200_ctx* ctx,
                                const void* src, const int64_t* src_off, const int32_t* src_len, const int32_t* dst_cap,
                                void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len,
                                int32_t n_blocks, int mode);

/* The same with src in device memory of the context's GPU (the offload of data that lives in HBM): the contract of
 * lz4b200_encode_batch_packed -- out_off[0..n], only the produced bytes land in dst (host memory, pageable or
 * page-locked), LZ4B200_E_ARG when dst_total_cap is too small -- plus that of every mixed call (MEM_DEVICE_TO_HOST above):
 * synchronous, ordered behind `stream`, no copy of src. */
int lz4b200_encode_batch_packed_from_device(lz4b200_ctx* ctx,
                                            const void* src, const int64_t* src_off, const int32_t* src_len,
                                            const int32_t* dst_cap, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                            int32_t* out_len, int32_t n_blocks, int mode, void* stream);

/* ---- offload without blocking: device memory <-> page-locked host memory, asynchronous on `stream` ------------------
 * The calls below do what their synchronous forms do -- lz4b200_encode_batch_packed_from_device,
 * lz4b200_decode_batch(LZ4B200_MEM_HOST_TO_DEVICE), lz4b200_decode_batch_packed_to_device, and the Wrap / Unwrap calls
 * between device and host memory -- with the same out_len, offsets and bytes, but only ENQUEUE their work on `stream` and
 * return without waiting for any device work: the thread that launches a model's kernels can offload a cache to host RAM,
 * or prefetch it back, and keep launching while the transfer runs.
 *   - Ordering: the call's device work runs after everything enqueued on `stream` before the call, and anything enqueued on
 *     `stream` after it sees all of its results.  Calls of one context are ordered among themselves on any streams.
 *   - Lifetime: the caller keeps src, dst, out_off and out_len alive and untouched until `stream` has passed the call (a
 *     cudaStreamSynchronize, or an event recorded behind it).  The offset, length and capacity arrays are host arrays
 *     read during the call only.
 *   - The host side is page-locked memory the device can address: cudaHostAlloc / cudaMallocHost, torch pin_memory(), or a
 *     lz4b200_host_register'd range.  Pageable memory, device memory, or memory without a device address there is
 *     LZ4B200_E_ARG.  out_off / out_len may be device memory of the context's GPU or page-locked host memory.
 *   - LZ4B200_E_ARG for a NULL argument, a negative length or memory of the wrong kind, before any device work.  A stream
 *     that is capturing a CUDA graph is LZ4B200_E_ARG before any CUDA work; the capture stays valid.
 *   - Never a wait on device work, except once when the context's buffers for these calls (or its HC arena) must grow: a
 *     call that needs no more than an earlier call of the same context never waits.
 *
 * encode_batch_packed_from_device_async: src is device memory of the context's GPU; dst is page-locked host memory.
 *   out_len[i] and out_off[0..n] (n_blocks+1 entries, out_off[n] the total) are written by the device and equal what
 *   lz4b200_encode_batch_packed_from_device gives for the same arguments; if out_off[n] <= dst_total_cap, dst[0, out_off[n])
 *   holds the same bytes.  A destination too small is still LZ4B200_OK (the total is known only on the device): out_off and
 *   out_len are filled, nothing outside [dst, dst + dst_total_cap) is written and the bytes inside it are unspecified, as in
 *   lz4b200_decode_batch_packed_to_device; the caller sees out_off[n] > dst_total_cap after synchronising.  n_blocks == 0 is
 *   LZ4B200_OK with out_off[0] = 0 written on the stream. */
int lz4b200_encode_batch_packed_from_device_async(lz4b200_ctx* ctx, const void* src, const int64_t* src_off,
                                                  const int32_t* src_len, const int32_t* dst_cap, void* dst,
                                                  int64_t dst_total_cap, int64_t* out_off, int32_t* out_len,
                                                  int32_t n_blocks, int mode, void* stream);
/* decode_batch_to_device_async: lz4b200_decode_batch(..., known_len, LZ4B200_MEM_HOST_TO_DEVICE, stream) without blocking.
 *   src is page-locked host memory; dst is device memory of the context's GPU.  out_len[i] and the bytes written equal what
 *   the synchronous call gives; nothing is written outside [dst_off[i], dst_off[i] + dst_cap[i]). */
int lz4b200_decode_batch_to_device_async(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                         void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len,
                                         int32_t n_blocks, int known_len, void* stream);
/* decode_batch_packed_to_device_async: lz4b200_decode_batch_packed_to_device without blocking.  src is page-locked host
 *   memory; dst is device memory of the context's GPU; out_off (n_blocks+1 entries) and out_len are written by the device.
 *   Results, bytes and the contract of a destination too small are those of the synchronous call.  n_blocks == 0 is
 *   LZ4B200_OK with out_off[0] = 0 written on the stream. */
int lz4b200_decode_batch_packed_to_device_async(lz4b200_ctx* ctx, const void* src, const int64_t* src_off,
                                                const int32_t* src_len, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                                int32_t* out_len, int32_t n_blocks, void* stream);

/* The same for Wrap packets (below), which describe themselves: a packet holds its raw length, so a batch restores from
 * the packet offsets alone, and an input that does not shrink is stored raw, so a packet is never above its input + 8
 * bytes whatever the data.
 *
 * wrap_batch_packed_from_device_async: lz4b200_wrap_batch_packed_from_device without blocking.  src is device memory of the
 *   context's GPU; dst is page-locked host memory.  out_off[0..n] (n+1 entries), out_len and the bytes equal what the
 *   synchronous call gives; sum(src_len[i] + 8) bytes of dst are always enough.  A destination too small is still
 *   LZ4B200_OK, as in lz4b200_encode_batch_packed_from_device_async: out_off and out_len are filled and nothing outside
 *   [dst, dst + dst_total_cap) is written.  A packet above INT32_MAX bytes (src_len[i] > INT32_MAX - 8) is LZ4B200_E_ARG.
 *   n == 0 is LZ4B200_OK with out_off[0] = 0 written on the stream. */
int lz4b200_wrap_batch_packed_from_device_async(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                                int high_compression, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                                int32_t* out_len, int32_t n, void* stream);
/* The two Unwraps from page-locked host memory read the packet headers on the DEVICE, from the bytes they stage, unlike the
 * synchronous ones, which read them on the host before any device work: the source may be written by work still queued on
 * `stream` when the call is made -- an asynchronous Wrap landing into the same buffer, for one -- and the host would read
 * what was there before.  The caller therefore needs only the packet offsets and lengths.
 *
 * unwrap_batch_to_device_async: lz4b200_unwrap_batch_to_device without blocking.  src is page-locked host memory; dst is
 *   device memory of the context's GPU.  out_len[i] equals what the synchronous call returns for the packet: bytes restored,
 *   LZ4B200_E_FORMAT or LZ4B200_E_ARG (a bad packet is that packet's status, never the call's).  Nothing is written outside
 *   [dst_off[i], dst_off[i] + dst_cap[i]). */
int lz4b200_unwrap_batch_to_device_async(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                         void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len,
                                         int32_t n, void* stream);
/* unwrap_batch_packed_to_device_async: unwrap into PACKED device output sized from the headers.  out_off[0..n] (n+1
 *   entries) = exclusive prefix sum of max(size, 0), size = the header's unwrapped size or the packet's negative status, is
 *   written by the device whether the total fits or not.
 *   - out_off[n] <= dst_total_cap: out_off, out_len and the bytes equal lz4b200_unwrap_batch_packed_to_device's.
 *   - out_off[n] > dst_total_cap: still LZ4B200_OK, under the contract of lz4b200_decode_batch_packed_to_device: nothing
 *     outside [dst, dst + dst_total_cap) is written, the bytes inside it are unspecified, and out_len[i] is non-negative
 *     exactly for the well-formed packets, where it equals the size.  This is weaker than the synchronous call's "dst is
 *     untouched", on purpose: the headers are read on the device a stage at a time, so the total is known only once the
 *     last stage has been staged, and holding the restored output back until then would take a second pass over the
 *     packets.  (A stage is restored when everything up to its end fits.  A packet whose header is well-formed but whose
 *     payload does not decode reports LZ4B200_E_FORMAT in a stage that was restored and its size in one that was not.)
 *   n == 0 is LZ4B200_OK with out_off[0] = 0 written on the stream. */
int lz4b200_unwrap_batch_packed_to_device_async(lz4b200_ctx* ctx, const void* src, const int64_t* src_off,
                                                const int32_t* src_len, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                                int32_t* out_len, int32_t n, void* stream);

/* Restoring from offsets that exist only on the device.  The packed asynchronous encode and Wrap write out_off on the
 * device, so the calls above, which read src_off / src_len on the host during the call, would make the caller wait for the
 * offload first.  The two calls below take src_off where the device reads it, when the call's work runs, so a whole
 * offload -> restore round trip is enqueued with no host wait: pass the offload's out_off as src_off, and its own
 * src_off / src_len as dst_off / dst_cap.
 *   - src is page-locked host memory, of which src_cap bytes may be read: nothing outside [src, src + src_cap) is read,
 *     whatever src_off holds, except the rest of an aligned 16-byte unit that overlaps the range (which lies in the same
 *     page-locked page).  src_off has n + 1 int64 entries, in device memory of the context's GPU or in page-locked host
 *     memory; block i spans [src_off[i], src_off[i+1]).  dst, dst_off, dst_cap and out_len are as in the host-offset form.
 *   - Each block's span may be at most a bound the host knows, by which the call sizes its stage buffers: a decode's
 *     lz4b200_compress_bound(dst_cap[i]); an Unwrap packet's dst_cap[i] + 8 (no packet that restores into dst_cap[i]
 *     bytes is larger).
 *   - A span is well-formed when 0 <= src_off[i] <= src_off[i+1] <= src_cap and its length is at most its bound.  Then
 *     out_len[i] and the bytes written equal what the host-offset form gives with src_len[i] = src_off[i+1] - src_off[i].
 *     Otherwise out_len[i] = LZ4B200_E_ARG, nothing of that block is read and nothing in its dst range is written.  This is
 *     where the two forms differ: a span longer than its bound (a packet with trailing bytes, for one) is rejected here
 *     but may be accepted by the host-offset form.
 *   - src_off[n] > src_cap means the offload that wrote the offsets did not fit its destination, so which of its bytes
 *     landed is unknown: every block is LZ4B200_E_ARG and dst is not written.  A destination sized by the offload's bound
 *     never hits this: sum(dst_cap) at compress_bound for an encode, sum(src_len + 8) for a Wrap.
 *   - The rest is the contract of the asynchronous calls above; the dst_off and dst_cap arrays are read during the call.
 *
 * decode_batch_to_device_at_async: lz4b200_decode_batch_to_device_async with the blocks' offsets read on the device.
 * unwrap_batch_to_device_at_async: lz4b200_unwrap_batch_to_device_async with the packets' offsets read on the device. */
int lz4b200_decode_batch_to_device_at_async(lz4b200_ctx* ctx, const void* src, int64_t src_cap, const int64_t* src_off,
                                            void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len,
                                            int32_t n_blocks, int known_len, void* stream);
int lz4b200_unwrap_batch_to_device_at_async(lz4b200_ctx* ctx, const void* src, int64_t src_cap, const int64_t* src_off,
                                            void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len,
                                            int32_t n, void* stream);

/* stream_decode_to_device_at_async: lz4b200_stream_decode_to_device_async (below) with the stream's size read on the device.
 * stream_encode_from_device_async writes the stream's size only on the device, and the host-walk decode needs it on the
 * host, so the caller would have to wait for the encode.  Here src_size (one int64, device memory of the context's GPU or
 * page-locked host memory) is read on the device when the call's work runs, and the chunk headers are walked there too:
 * pass the encode's out_size as src_size and enqueue the whole round trip with no host wait,
 *     stream_encode_from_device_async(x, n, B, hc, buf, stream_bound(n, B), d_size, s)
 *     stream_decode_to_device_at_async(buf, stream_bound(n, B), d_size, B, y, n, d_out, s)
 *   - src is page-locked host memory of which src_cap bytes may be read; block_size is the largest rawLen a chunk may have
 *     (the chunk size the stream was written with); dst is device memory of the context's GPU, dst_cap its bytes.  src may
 *     be null when src_cap == 0, dst when dst_cap == 0.  Any other null pointer, src_cap < 0, dst_cap < 0 or block_size
 *     outside [1, INT32_MAX - 11] returns LZ4B200_E_ARG and enqueues nothing.
 *   - Let S = *src_size and K = ceil(dst_cap / block_size), the chunk count of a stream of dst_cap bytes at block_size.  S < 0
 *     or S > src_cap: *out_size = LZ4B200_E_ARG, nothing of src is read and dst is not written.  Otherwise the chunks of
 *     src[0, S) are walked in order with exactly the rules of the host walk; the first of these ends it: a malformed header
 *     (LZ4B200_E_FORMAT), a chunk with rawLen > block_size, a (K+1)-th chunk (empty chunks count), or a chunk whose output
 *     would end past dst_cap (each LZ4B200_E_ARG).  Else *out_size = LZ4B200_E_FORMAT when a compressed chunk does not
 *     decode from exactly its compLen bytes, and otherwise the decoded size T, with dst[0, T) what
 *     lz4b200_stream_decode_to_device writes for src[0, S).
 *   - So for every well-formed stream whose chunks keep the three bounds, and for a malformed one whose chunks before the
 *     first malformed header keep them, *out_size equals what lz4b200_stream_decode_to_device(src, S, dst, dst_cap)
 *     returns.  The bounds are where the two differ, as the block calls' span bound above: the host sizes the stages'
 *     buffers before the device has seen a header.
 *   - Nothing outside [dst, dst + dst_cap) is written; after a failure the bytes inside it are unspecified.  Nothing outside
 *     [src, src + S) is read, except the rest of an aligned 16-byte unit that overlaps it.
 *   - The rest is the contract of the asynchronous calls.  The call holds no per-chunk host metadata; its device work
 *     grows with K, since the host cuts the stages before the size is known. */
int lz4b200_stream_decode_to_device_at_async(lz4b200_ctx* ctx, const void* src, int64_t src_cap, const int64_t* src_size,
                                             int32_t block_size, void* dst, int64_t dst_cap, int64_t* out_size,
                                             void* stream);

/* Compaction of fixed-stride encoder slots into one contiguous payload (device memory only): the batched form of
 * the Buffer.BlockCopy trim in LZ4Codec.Encode (src/LZ4/LZ4Codec.cs:357-364).  out_off[i] (int64, n_blocks+1
 * entries) = exclusive prefix sum of max(len[i],0); block i's bytes are copied to packed + out_off[i]. */
int lz4b200_compact(lz4b200_ctx* ctx, const void* slots, const int64_t* slot_off, const int32_t* len,
                    void* packed, int64_t* out_off, int32_t n_blocks, void* stream);

/* ---- CUDA graphs: capturing the device-memory calls -------------------------------------------------------------
 * The device-memory entry points -- lz4b200_encode_batch / decode_batch / measure_batch with LZ4B200_MEM_DEVICE,
 * decode_batch_packed, compact, wrap_batch_device, unwrap_batch_device, unwrap_batch_packed and synth_fill -- may be
 * enqueued on a stream that is capturing a CUDA graph, in any capture mode:
 *   - Replaying the graph does exactly what the same call would do enqueued on the replay stream at replay time: the same
 *     kernels, byte-identical outputs, the same out_len and out_off, for whatever the captured input buffers hold then.
 *     The pointers and n_blocks are fixed at capture.
 *   - Captured calls, eager calls and replays of graphs of one context, on any streams, stay ordered on the context's
 *     shared scratch in host enqueue order, as eager calls are (one HC encode at a time, one user of the scan scratch,
 *     capacities and packet view at a time).  Graphs that hold calls of one context may be replayed concurrently.
 *     Calls of one capture that the capture forks onto several streams are ordered too, as long as one thread at a
 *     time captures calls of the context (one context per caller thread, as above).
 *   - A captured call never allocates, frees or synchronises.  When the context's scratch is too small for it, or its
 *     4096 counter sets for captured calls are used up, it returns LZ4B200_E_ARG, enqueues nothing and leaves the
 *     capture valid; lz4b200_last_error() says what is missing.  Call lz4b200_reserve before capturing.
 *   - Scratch that a captured call referenced is never freed before lz4b200_destroy: a later growth (an eager call, or
 *     lz4b200_reserve, or set_option("hc_concurrency")) allocates a new buffer and keeps the old one.  A context that
 *     never captured frees and grows its scratch as before; every context holds the 64 KiB of counter sets.  Do not
 *     replay a graph after lz4b200_destroy of a context it holds calls of.
 *   - lz4b200_launch_count counts the launches a call enqueues when it is captured, not replays.
 * Every other call that takes a `stream` synchronises with the host (the mixed-memory batches, the packed encode from
 * and decode to device memory, the LZ4Stream and the Wrap / Unwrap calls between device and host memory): on a capturing
 * stream it returns LZ4B200_E_ARG before any CUDA work, and the capture stays valid.  So do the asynchronous calls --
 * lz4b200_encode_batch_packed_from_device_async, decode_batch_to_device_async, decode_batch_packed_to_device_async,
 * wrap_batch_packed_from_device_async, unwrap_batch_to_device_async, unwrap_batch_packed_to_device_async,
 * decode_batch_to_device_at_async, unwrap_batch_to_device_at_async,
 * stream_encode_from_device_async, stream_decode_to_device_async and stream_decode_to_device_at_async -- which do not
 * synchronise but share the context's stage buffers between eager calls and, all but the stream encode and the stream
 * decode from a device-read size, hand the device host metadata that a graph would have to keep alive.  lz4b200_peer_copy is not covered.
 * The calls without a stream (host-memory batches, single-block functions, lz4b200_synchronize, lz4b200_reserve) use
 * the legacy default stream or synchronise the device: they must not be made while any thread of the process captures
 * in cudaStreamCaptureModeGlobal.
 *
 * reserve: grows, eagerly, every piece of device scratch a device-memory call of at most max_blocks blocks takes; with
 * high_compression != 0 also the HC state arena, as an HC device batch of max_blocks blocks sizes it under the current
 * "hc_kernel", "hc_warps_per_sm" and "hc_concurrency" (changing those later may need more).  Afterwards any such call can
 * be captured.  LZ4B200_E_ARG for a NULL context or max_blocks < 0. */
int lz4b200_reserve(lz4b200_ctx* ctx, int32_t max_blocks, int high_compression);

/* ---- single-block entry points (host pointers), 1:1 with the reference's native API -------------------------- */
/* original/lz4.h:59-60  LZ4_compress_limitedOutput */
int lz4b200_compress_limitedOutput(const char* source, char* dest, int isize, int maxOutputSize);
/* original/lz4hc.h:57   LZ4_compressHC_limitedOutput */
int lz4b200_compressHC_limitedOutput(const char* source, char* dest, int isize, int maxOutputSize);
/* original/lz4.h:101    LZ4_uncompress.  `isize` (the compressed length every managed caller holds,
 * src/LZ4pn/LZ4Codec.Unsafe.cs:366-371) is added because the bytes must be staged to the device; reads never pass it. */
int lz4b200_uncompress(const char* source, char* dest, int isize, int osize);
/* original/lz4.h:116    LZ4_uncompress_unknownOutputSize */
int lz4b200_uncompress_unknownOutputSize(const char* source, char* dest, int isize, int maxOutputSize);

/* ---- framing built on the batch calls ("next" rows of SURVEY.md 8f) ------------------------------------------
 * LZ4Stream chunk format (src/LZ4/LZ4Stream.cs:239-312): varint(flags) varint(rawLen) [varint(compLen)] payload.
 * stream_encode cuts `src` into block_size chunks, encodes all of them in one batch and writes the exact byte
 * stream an LZ4Stream(..., Compress, highCompression, block_size) would have produced for one Write + Close.
 * Returns bytes written, or a negative status (LZ4B200_E_ARG if dst_cap is too small / the stream is malformed).
 * The frames are written on the device, where a chunk's frame must fit an int32: a stream that holds a chunk above
 * INT32_MAX - 11 bytes (min(block_size, n) > INT32_MAX - 11) is LZ4B200_E_ARG.  Any block_size works below that. */
int64_t lz4b200_stream_bound(int64_t n, int32_t block_size);
int64_t lz4b200_stream_encode(lz4b200_ctx* ctx, const void* src, int64_t n, int32_t block_size, int high_compression,
                              void* dst, int64_t dst_cap);
int64_t lz4b200_stream_decoded_size(const void* src, int64_t n);     /* sum of rawLen over all chunks, <0 = malformed */
int64_t lz4b200_stream_decode(lz4b200_ctx* ctx, const void* src, int64_t n, void* dst, int64_t dst_cap);

/* The same stream between device memory and host memory: the stream bytes stay in host memory (a file, a socket), the
 * raw bytes in HBM, and only the stream bytes cross PCIe, once, overlapped with the kernels.  The host walks the chunk
 * headers; the device encodes, decodes, writes the frames and copies stored payloads.  Both follow the contract of every
 * mixed call (LZ4B200_MEM_DEVICE_TO_HOST above): synchronous, ordered behind the work already queued on `stream`, and
 * LZ4B200_E_ARG when either side is the wrong kind of memory.  n == 0 returns 0.
 *
 * stream_encode_from_device: the wire bytes lz4b200_stream_encode writes for a host copy of src.  src: device memory of
 *   the context's GPU (n bytes); dst: host memory, pageable or page-locked, dst_cap >= lz4b200_stream_bound(n, block_size).
 *   block_size >= 1 and at most INT32_MAX - 11 (a chunk's frame fits an int32).  Returns bytes written or a negative status. */
int64_t lz4b200_stream_encode_from_device(lz4b200_ctx* ctx, const void* src, int64_t n, int32_t block_size,
                                          int high_compression, void* dst, int64_t dst_cap, void* stream);
/* stream_decode_to_device: the decoded stream, lz4b200_stream_decoded_size bytes, at dst (device memory of the context's
 *   GPU).  src: host memory.  Returns the decoded size or a negative status: LZ4B200_E_FORMAT / E_ARG exactly where
 *   lz4b200_stream_decode returns them.  Nothing is written outside [dst, dst + decoded size); a malformed header is found
 *   before any device work, so nothing is written at all; after a chunk that does not decode (E_FORMAT) the bytes inside
 *   the range are unspecified. */
int64_t lz4b200_stream_decode_to_device(lz4b200_ctx* ctx, const void* src, int64_t n, void* dst, int64_t dst_cap,
                                        void* stream);

/* The same stream between device memory and PAGE-LOCKED host memory without blocking: the contract of the asynchronous
 * calls above ("offload without blocking": ordering on `stream` and among the context's calls, lifetime, page-locked host
 * side, refusal of a capturing stream, no wait on device work except once when the context's buffers or HC arena grow).
 * out_size may be device memory of the context's GPU or page-locked host memory; it is written by the device.  Argument
 * and memory checks return what the synchronous calls return wherever the host can decide them.  One pointer and one
 * length describe the whole offload: the bytes can be written to a file or a socket afterwards and read by any LZ4Stream.
 *
 * stream_encode_from_device_async: src is n bytes of device memory of the context's GPU; dst is page-locked host memory,
 *   dst_cap >= lz4b200_stream_bound(n, block_size), so the stream always fits.  *out_size and dst[0, *out_size) equal what
 *   lz4b200_stream_encode_from_device returns and writes for the same arguments; nothing outside [dst, dst + *out_size) is
 *   written.  block_size >= 1 and at most INT32_MAX - 11, as in the synchronous call.  n == 0 writes *out_size = 0 on the
 *   stream.  The call's page-locked metadata is O(pipeline stages): a stage's chunk table is computed on the device.
 * stream_decode_to_device_async: src is the n bytes of a whole stream in page-locked host memory; dst is device memory of
 *   the context's GPU.  The HOST walks the chunk headers during the call, as the synchronous call does: a caller who can
 *   pass n has the stream's bytes in place (an asynchronous encode reports its size only on the device), so src must hold
 *   the whole stream when the call is made, and stay untouched until `stream` has passed the call.
 *   - A malformed header returns LZ4B200_E_FORMAT, and dst_cap below the decoded size LZ4B200_E_ARG; either way nothing is
 *     enqueued and neither dst nor out_size is written.
 *   - Otherwise the device writes *out_size: the decoded size, or LZ4B200_E_FORMAT when a compressed chunk does not decode
 *     from exactly its compLen bytes (where the synchronous call returns LZ4B200_E_FORMAT).  Nothing is written outside
 *     [dst, dst + decoded size); after a chunk that fails, the bytes inside it are unspecified.
 *   - n == 0, or a stream of empty chunks, writes *out_size = 0 on the stream.
 *   The call's page-locked metadata is O(non-empty chunks): one entry each (payload offset, compLen, rawLen, stored flag,
 *   output offset), held until `stream` has passed the call. */
int lz4b200_stream_encode_from_device_async(lz4b200_ctx* ctx, const void* src, int64_t n, int32_t block_size,
                                            int high_compression, void* dst, int64_t dst_cap, int64_t* out_size,
                                            void* stream);
int lz4b200_stream_decode_to_device_async(lz4b200_ctx* ctx, const void* src, int64_t n, void* dst, int64_t dst_cap,
                                          int64_t* out_size, void* stream);

/* LZ4Codec.Wrap / Unwrap packet (src/LZ4/LZ4Codec.cs:510-543,574-599): u32le rawLen, u32le storedLen, payload. */
int lz4b200_wrap(lz4b200_ctx* ctx, const void* src, int32_t n, int high_compression, void* dst, int32_t dst_cap);
int lz4b200_unwrap_size(const void* src, int32_t n);
int lz4b200_unwrap(lz4b200_ctx* ctx, const void* src, int32_t n, void* dst, int32_t dst_cap);

/* The same for n packets at once: ONE encode / decode batch instead of one H2D + launch + D2H per packet.  Packet i is
 * byte for byte what lz4b200_wrap makes of input i.  wrap_batch: dst_cap[i] >= src_len[i] + 8; out_len[i] = packet size.
 * unwrap_batch: dst_cap[i] >= lz4b200_unwrap_size(packet i); out_len[i] = bytes restored or a negative status. */
int lz4b200_wrap_batch(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len, int high_compression,
                       void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n);
int lz4b200_unwrap_batch(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                         void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len, int32_t n);

/* The same packets in device memory, asynchronous on `stream` (no host synchronisation, except that an HC batch may
 * synchronise once to grow the context's HC arena, as device HC batches do).  A batch already in HBM never crosses PCIe:
 * the encoders / decoders run as in lz4b200_{encode,decode}_batch(MEM_DEVICE), and the header, the stored-raw rule and
 * the stored copies run on the device.  Packets and statuses are byte for byte those of the host calls above, so a packet
 * made on either side, or by lz4net's LZ4Codec.Wrap / WrapHC, is read by the other's Unwrap.
 *
 * wrap_batch_device: packet i = Wrap / WrapHC of src + src_off[i] (src_len[i] bytes), written at dst + dst_off[i];
 *   dst_cap[i] >= src_len[i] + 8.  out_len[i] = packet size (at most src_len[i] + 8), or LZ4B200_E_ARG for that packet
 *   (negative length, capacity too small), which then has nothing written.  Bytes behind out_len[i] in the slot may be
 *   overwritten.  For packets back to back, pass the slots and out_len to lz4b200_compact. */
int lz4b200_wrap_batch_device(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                              int high_compression, void* dst, const int64_t* dst_off, const int32_t* dst_cap,
                              int32_t* out_len, int32_t n, void* stream);
/* unwrap_batch_device: packet i = src + src_off[i], src_len[i] bytes, restored to dst + dst_off[i], capacity dst_cap[i].
 *   out_len[i] = bytes restored, LZ4B200_E_FORMAT or LZ4B200_E_ARG: what lz4b200_unwrap_batch returns for the same packet
 *   and capacity.  Nothing is written outside [dst_off[i], dst_off[i] + dst_cap[i]). */
int lz4b200_unwrap_batch_device(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len,
                                int32_t n, void* stream);
/* unwrap_batch_packed: unwrap into PACKED output that the library sizes from the headers, with the contract of
 * lz4b200_decode_batch_packed: out_off[0..n] (int64, n+1 entries) = exclusive prefix sum of max(size, 0), size = the
 * header's unwrapped size or the packet's negative status.  If out_off[n] <= dst_total_cap, packet i is restored to
 * dst + out_off[i] and out_len[i] is as in unwrap_batch_device; otherwise dst is untouched and out_len holds the sizes. */
int lz4b200_unwrap_batch_packed(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len,
                                int32_t n, void* stream);

/* The same packets between device memory and host memory: the packets stay in host memory (a socket buffer, an RPC
 * payload), the raw bytes in HBM, and only the packets cross PCIe, once, overlapped with the kernels.  The host reads the
 * unwrap headers; the device encodes, decodes, writes the headers and copies stored payloads.  Offsets, lengths, out_off
 * and out_len are host arrays.  All four follow the contract of every mixed call (LZ4B200_MEM_DEVICE_TO_HOST above):
 * synchronous, ordered behind the work already queued on `stream`, and LZ4B200_E_ARG when either side is the wrong kind
 * of memory.  n == 0 is LZ4B200_OK (the packed forms set out_off[0] = 0).
 *
 * wrap_batch_from_device: src in device memory of the context's GPU, dst in host memory, pageable or page-locked.  Packet
 *   i is byte for byte what lz4b200_wrap_batch makes of a host copy of input i; it lands at dst + dst_off[i], and only
 *   its out_len[i] bytes are written there.  As in lz4b200_wrap_batch, a negative length or dst_cap[i] < src_len[i] + 8
 *   makes the whole call LZ4B200_E_ARG before any device work. */
int lz4b200_wrap_batch_from_device(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                   int high_compression, void* dst, const int64_t* dst_off, const int32_t* dst_cap,
                                   int32_t* out_len, int32_t n, void* stream);
/* wrap_batch_packed_from_device: the same packets back to back in host memory, in packet order (what a sender writes to
 *   a socket): packet i at dst + out_off[i], out_off[0..n] (n+1 entries), out_off[n] the total.  sum(src_len[i] + 8) is
 *   always enough; a smaller dst_total_cap that the packets do not fit is LZ4B200_E_ARG, as in
 *   lz4b200_encode_batch_packed_from_device.  A packet above INT32_MAX bytes (src_len[i] > INT32_MAX - 8) is E_ARG. */
int lz4b200_wrap_batch_packed_from_device(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                          int high_compression, void* dst, int64_t dst_total_cap, int64_t* out_off,
                                          int32_t* out_len, int32_t n, void* stream);
/* unwrap_batch_to_device: packets in host memory, outputs in device memory of the context's GPU.  out_len[i] is what
 *   lz4b200_unwrap_batch returns for the same packet and capacity: bytes restored, LZ4B200_E_FORMAT or E_ARG (a bad packet
 *   is that packet's status, never the call's).  Nothing is written outside [dst_off[i], dst_off[i] + dst_cap[i]). */
int lz4b200_unwrap_batch_to_device(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                   void* dst, const int64_t* dst_off, const int32_t* dst_cap, int32_t* out_len,
                                   int32_t n, void* stream);
/* unwrap_batch_packed_to_device: the contract of lz4b200_unwrap_batch_packed with out_off and out_len on the host.  The
 *   sizes come from the headers before any device work; if out_off[n] > dst_total_cap, dst is untouched and out_len holds
 *   the sizes, otherwise it is unwrap_batch_to_device with dst_off = out_off and dst_cap = the sizes. */
int lz4b200_unwrap_batch_packed_to_device(lz4b200_ctx* ctx, const void* src, const int64_t* src_off, const int32_t* src_len,
                                          void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len,
                                          int32_t n, void* stream);

/* ---- host buffers the caller keeps for a while (a pinned byte[] behind a GCHandle, a native arena) --------------------
 * Host-memory batches copy straight from / to the caller's buffers.  From pageable memory the driver stages every copy
 * through its own pinned bounce buffers, synchronously; page-locking a long-lived buffer once (cudaHostRegister) lets the
 * same calls run at the full pipelined rate.  Optional: everything works without it. */
int lz4b200_host_register(void* ptr, int64_t bytes);
int lz4b200_host_unregister(void* ptr);

/* ---- one stream, several GPUs of one node (BASELINE configs[3]; lz4net_b200/shard.py StreamWindow) --------------------
 * Asynchronous copy between device buffers of two GPUs (either side may be memory another process exported with CUDA
 * IPC), ordered on `stream` of the CURRENT device, executed by the copy engines over NVLink -- it overlaps codec kernels,
 * which a send/recv kernel of a communication library does not.  Enables peer access on first use. */
int lz4b200_peer_copy(void* dst, const void* src, int64_t bytes, void* stream);

/* ---- synthetic workload generator (bench/test utility; device memory) ----------------------------------------
 * Fills n_blocks * block_size bytes at dst with entropy class cls (0 E0, 1 E50, 2 E100, 3 ETEXT), block index
 * first_block + i, exactly as lz4net_b200/synth.py defines them. */
int lz4b200_synth_fill(lz4b200_ctx* ctx, void* dst, int64_t n_blocks, int32_t block_size, int cls, uint64_t seed,
                       int64_t first_block, void* stream);

/* Tuning knobs (bench / profiling only).  key: "decode_lanes" (4|8|16|32 lanes per block, +100 = the output-staged
 * variant; 1 = the lane-per-block decoder), "decode_lanes_auto" (the decoder is
 * picked per batch from the compression ratio: the default), "encode_ctas_per_sm" (encoder warps = blocks in
 * flight per SM, 0 = as many as shared memory allows: 14), "encode_variant" (1 = always exact same-hash votes, 2 = resolved
 * through the table: default),
 * "encode_prefetch" (bytes of input kept prefetched ahead of the parse; 0 off, < 0 L2 only), "encode_lane_copy_max" /
 * "encode_probe_max" / "encode_wide_min" (path-selection heuristics of the fast encoder, lz4_encode.cuh EncTune: they
 * never change the emitted bytes), "hc_kernel" (which LZ4HC kernel encodes a batch: -1 = chosen per batch, the default -- at most
 * three blocks per SM: kernel 1, larger batches: kernel 2; 0 = one thread per block, any block size; 1 / 2 = one warp per
 * block: blocks of at most 64 KiB on a static index of the block's hash buckets -- 1 stages the block in shared memory, 2
 * reads it through L1 -- and larger blocks, with either value, over a sliding 64 KiB window of index segments; the rare
 * block whose chains depend on the parse goes to kernel 0 inside the same call), "hc_warps_per_sm" (kernels 1 / 2: blocks of at most 64 KiB in flight per SM,
 * 0 = the default: 3 / 32),
 * "hc_concurrency" (kernel 0: blocks in flight), "host_chunk_mb" (bytes per pipeline stage of host-memory batches).
 * Returns LZ4B200_OK or LZ4B200_E_ARG. */
int lz4b200_set_option(lz4b200_ctx* ctx, const char* key, int64_t value);
/* The current value of an integer option ("hc_kernel", "hc_warps_per_sm", "hc_concurrency", "decode_lanes",
 * "encode_variant", "encode_ctas_per_sm").  Returns LZ4B200_OK or LZ4B200_E_ARG. */
int lz4b200_get_option(lz4b200_ctx* ctx, const char* key, int64_t* value);

/* Kernel launches issued through this context since creation (bench.py reports it as gpu_launches). */
int64_t lz4b200_launch_count(lz4b200_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* LZ4B200_H */
