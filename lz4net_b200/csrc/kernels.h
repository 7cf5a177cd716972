// kernels.h -- internal launcher interface between the C-ABI translation unit and the kernel translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lz4b200 {

struct BatchArgs {
    const uint8_t* src; const int64_t* src_off; const int32_t* src_len;
    uint8_t* dst; const int64_t* dst_off; const int32_t* dst_cap;
    int32_t* out_len; int32_t n_blocks;
};

struct DeviceInfo { int num_sms; int smem_per_sm; int smem_optin; };

// All launchers are asynchronous on `stream`; `counter` is a device uint32 the launcher zeroes itself (dynamic
// block hand-out).  They return the launch error (cudaSuccess on success) and add to *launches.
// lanes_per_block: 32 | 16 | 8 | 4 (+100 = output-staged), 1 | 2 = the lane-per-block decoder, 0 = chosen on the device from
// the batch's compression ratio.  `counter` points at FOUR device words the launcher owns (block counter, pick, two more counters).
int         decode_lanes_for_ratio(double ratio);
// gate (optional): a device int; when it reads 0 at run time every decoder kernel of the launch returns at once.
cudaError_t launch_decode(const BatchArgs& a, bool known_len, int lanes_per_block, uint32_t* counter,
                          const DeviceInfo& dev, cudaStream_t stream, int64_t* launches, const int* gate = nullptr);
// out_len[i] = what launch_decode would store for block i, nothing else is written (a.dst / a.dst_off unused; a.dst_cap
// may be null when !known_len: INT32_MAX for every block).
cudaError_t launch_measure(const BatchArgs& a, bool known_len, const DeviceInfo& dev, cudaStream_t stream, int64_t* launches);
// cap[i] = max(size[i], 0); *fits = out_off[n] <= total_cap.  A stage of the host pipeline (lz4_packed.cuh) also passes
// base_in (the running total of the earlier stages; null = 0), abs_off (abs_off[i] = base + out_off[i]) and total_out
// (receives base + out_off[n]; a cell other than base_in); *fits is then base + out_off[n] <= total_cap.
cudaError_t launch_packed_prep(const int32_t* size, const int64_t* out_off, int32_t n, int64_t total_cap, int32_t room, int32_t* cap,
                               int* fits, cudaStream_t stream, int64_t* launches, const int64_t* base_in = nullptr,
                               int64_t* abs_off = nullptr, int64_t* total_out = nullptr);
cudaError_t launch_encode_fast(const BatchArgs& a, uint32_t* counter, int warps_per_sm, const int* tune4 /* prefetch, lane_copy_max, probe_max, wide_min */, int variant,
                               const DeviceInfo& dev, cudaStream_t stream, int64_t* launches);
size_t      hc_scratch_bytes(int concurrency);
cudaError_t launch_encode_hc(const BatchArgs& a, void* scratch, int concurrency, uint32_t* counter,
                             const DeviceInfo& dev, cudaStream_t stream, int64_t* launches);
// one warp per block on a static index for blocks <= 64 KiB (variant 1: the block staged in shared memory, <= 3 warps per
// SM; 2: nothing in shared memory, <= 32 warps per SM), then one warp per block over a sliding 64 KiB window for the blocks
// above 64 KiB, then the thread-per-block kernel over whatever is still handed back.  n_large = the number of blocks above
// 64 KiB, -1 = not known (device-memory batches: the arena is sized as if every block were one).
size_t      hcw_scratch_bytes(int32_t n_blocks, int32_t n_large, int variant, int warps_per_sm, const DeviceInfo& dev);
cudaError_t launch_encode_hcw(const BatchArgs& a, void* scratch, int variant, int warps_per_sm, int32_t n_large, uint32_t* counter,
                              const DeviceInfo& dev, cudaStream_t stream, int64_t* launches);
// kernel chosen per batch: small batches -> the shared-memory warp kernel, larger ones -> the one with nothing in shared
// memory (`counter` = four words)
size_t      hc_auto_scratch_bytes(int32_t n_blocks, int32_t n_large, const DeviceInfo& dev);
cudaError_t launch_encode_hc_auto(const BatchArgs& a, void* scratch, int32_t n_large, uint32_t* counter,
                                  const DeviceInfo& dev, cudaStream_t stream, int64_t* launches);
cudaError_t launch_compact(const uint8_t* slots, const int64_t* slot_off, const int32_t* len, uint8_t* packed,
                           int64_t* out_off, int32_t n_blocks, void* scan_tmp, size_t scan_tmp_bytes,
                           const DeviceInfo& dev, cudaStream_t stream, int64_t* launches);
size_t      compact_tmp_bytes(int32_t n_blocks);
// Wrap / Unwrap packets in device memory (wrap.cu, lz4_wrap.cuh).  The scratch holds the codec's view of the batch: payload
// offsets, lengths and capacities per packet, and the codec's per-packet results.
struct WrapScratch { int64_t* off; int32_t* len; int32_t* cap; int32_t* res; };
// a = the caller's batch (src_off / src_len / dst_off / dst_cap / out_len of the packets)
cudaError_t launch_wrap_prep(const BatchArgs& a, const WrapScratch& w, cudaStream_t stream, int64_t* launches);
cudaError_t launch_wrap_finish(const BatchArgs& a, const WrapScratch& w, cudaStream_t stream, int64_t* launches);
// a.dst_cap may be null (no limit: the packed unwrap); out_len[i] = the packet's size or status until the finish step
cudaError_t launch_unwrap_prep(const BatchArgs& a, const WrapScratch& w, cudaStream_t stream, int64_t* launches);
// gate (optional): a device int; when it reads 0 the kernel returns at once
cudaError_t launch_unwrap_finish(const BatchArgs& a, const WrapScratch& w, const int* gate, cudaStream_t stream, int64_t* launches);
// LZ4Stream frames in device memory (stream.cu, lz4_stream.cuh).  a = the encoded batch: src / src_off / src_len = the
// chunks' raw bytes, dst / dst_off = the encoder's slots, out_len = its results.  frame_len[i] = the size of chunk i's
// frame; launch_stream_frame writes frame i at frames + frame_off[i].
cudaError_t launch_stream_frame_size(const BatchArgs& a, int32_t* frame_len, cudaStream_t stream, int64_t* launches);
cudaError_t launch_stream_frame(const BatchArgs& a, bool hc, uint8_t* frames, const int64_t* frame_off, cudaStream_t stream,
                                int64_t* launches);
// a = the decoded batch (src / src_off = the staged stream and the payload offsets, dst / dst_off = the output): copies
// stored_len[i] bytes of payload i to its output; entries with stored_len[i] == 0 do nothing
cudaError_t launch_stream_stored(const BatchArgs& a, const int32_t* stored_len, cudaStream_t stream, int64_t* launches);
cudaError_t launch_synth(uint8_t* dst, int64_t n_blocks, int32_t block_size, int cls, uint64_t seed, int64_t first_block,
                         const DeviceInfo& dev, cudaStream_t stream, int64_t* launches);

}  // namespace lz4b200
