// stream.cu -- kernels + launchers of the LZ4Stream frame steps in device memory (see lz4_stream.cuh for the rules).
#include "../../include/lz4b200.h"
#include "kernels.h"
#include "lz4_stream.cuh"

namespace lz4b200 {

constexpr int SIZE_THREADS = 256;
constexpr int COPY_THREADS = 256;                      // 8 chunks per CTA, a warp each
constexpr int COPY_WARPS = COPY_THREADS / 32;

static unsigned size_grid(int32_t n) { return (unsigned)(((int64_t)n + SIZE_THREADS - 1) / SIZE_THREADS); }
static unsigned copy_grid(int32_t n) { return (unsigned)(((int64_t)n + COPY_WARPS - 1) / COPY_WARPS); }

__global__ void __launch_bounds__(SIZE_THREADS)
lz4_stream_frame_size_kernel(const int32_t* raw_len, const int32_t* res, int32_t n, int32_t* frame_len)
{
    const int64_t i = (int64_t)blockIdx.x * SIZE_THREADS + threadIdx.x;
    if (i < n) frame_len[i] = stream_frame_size(raw_len[i], res[i]);
}

__global__ void __launch_bounds__(COPY_THREADS)
lz4_stream_frame_kernel(const uint8_t* src, const int64_t* src_off, const int32_t* raw_len, const uint8_t* comp,
                        const int64_t* comp_off, const int32_t* res, int32_t n, bool hc, uint8_t* frames, const int64_t* frame_off)
{
    const int64_t i = (int64_t)blockIdx.x * COPY_WARPS + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = (int)(threadIdx.x & 31);
    stream_frame_one(src + src_off[i], raw_len[i], comp + comp_off[i], res[i], hc, frames + frame_off[i], lane);
}

__global__ void __launch_bounds__(COPY_THREADS)
lz4_stream_stored_kernel(const uint8_t* src, const int64_t* src_off, const int32_t* stored_len, uint8_t* dst,
                         const int64_t* dst_off, int32_t n)
{
    const int64_t i = (int64_t)blockIdx.x * COPY_WARPS + (threadIdx.x >> 5);
    if (i >= n) return;
    stream_stored_one(src + src_off[i], stored_len[i], dst + dst_off[i], (int)(threadIdx.x & 31));
}

__global__ void __launch_bounds__(SIZE_THREADS)
lz4_stream_cut_kernel(int64_t first, int32_t m, int32_t block_size, int64_t n, int64_t* so, int32_t* len, int64_t* dof, int32_t* cap)
{
    const int64_t i = (int64_t)blockIdx.x * SIZE_THREADS + threadIdx.x;
    if (i < m) stream_cut_one(i, first, block_size, n, so, len, dof, cap);
}

// Every failing entry stores 1; nothing stores 0, so the racing stores agree.
__global__ void __launch_bounds__(SIZE_THREADS)
lz4_stream_status_kernel(const int32_t* comp_len, const int32_t* stored, const int32_t* res, int32_t m, int* failed)
{
    const int64_t i = (int64_t)blockIdx.x * SIZE_THREADS + threadIdx.x;
    if (i < m && stream_chunk_failed(stored[i], comp_len[i], res[i])) *failed = 1;
}

__global__ void lz4_stream_result_kernel(const int* failed, int64_t total, int64_t* out_size)
{
    *out_size = *failed ? (int64_t)LZ4B200_E_FORMAT : total;
}

// One warp walks a stage's headers: the walk is a chain of dependent reads of host memory.
__global__ void __launch_bounds__(32) lz4_stream_walk_kernel(const StreamWalkStage w)
{
    stream_walk_stage(w, (int)threadIdx.x);
}

__global__ void lz4_stream_walk_result_kernel(const int* failed, const int64_t* carry, int64_t* out_size)
{
    *out_size = stream_walk_result(carry, *failed);
}

cudaError_t launch_stream_cut(int64_t first, int32_t m, int32_t block_size, int64_t n, int64_t* so, int32_t* len, int64_t* dof,
                              int32_t* cap, cudaStream_t stream, int64_t* launches)
{
    if (m <= 0) return cudaSuccess;
    lz4_stream_cut_kernel<<<size_grid(m), SIZE_THREADS, 0, stream>>>(first, m, block_size, n, so, len, dof, cap);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_stream_status(const int32_t* comp_len, const int32_t* stored, const int32_t* res, int32_t m, int* failed,
                                 cudaStream_t stream, int64_t* launches)
{
    if (m <= 0) return cudaSuccess;
    lz4_stream_status_kernel<<<size_grid(m), SIZE_THREADS, 0, stream>>>(comp_len, stored, res, m, failed);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_stream_result(const int* failed, int64_t total, int64_t* out_size, cudaStream_t stream, int64_t* launches)
{
    lz4_stream_result_kernel<<<1, 1, 0, stream>>>(failed, total, out_size);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_stream_walk(const StreamWalkStage& w, cudaStream_t stream, int64_t* launches)
{
    lz4_stream_walk_kernel<<<1, 32, 0, stream>>>(w);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_stream_walk_result(const int* failed, const int64_t* carry, int64_t* out_size, cudaStream_t stream, int64_t* launches)
{
    lz4_stream_walk_result_kernel<<<1, 1, 0, stream>>>(failed, carry, out_size);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_stream_frame_size(const BatchArgs& a, int32_t* frame_len, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    lz4_stream_frame_size_kernel<<<size_grid(a.n_blocks), SIZE_THREADS, 0, stream>>>(a.src_len, a.out_len, a.n_blocks, frame_len);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_stream_frame(const BatchArgs& a, bool hc, uint8_t* frames, const int64_t* frame_off, cudaStream_t stream,
                                int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    lz4_stream_frame_kernel<<<copy_grid(a.n_blocks), COPY_THREADS, 0, stream>>>(a.src, a.src_off, a.src_len, a.dst, a.dst_off,
                                                                               a.out_len, a.n_blocks, hc, frames, frame_off);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_stream_stored(const BatchArgs& a, const int32_t* stored_len, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    lz4_stream_stored_kernel<<<copy_grid(a.n_blocks), COPY_THREADS, 0, stream>>>(a.src, a.src_off, stored_len, a.dst, a.dst_off,
                                                                                a.n_blocks);
    if (launches) ++*launches;
    return cudaGetLastError();
}

}  // namespace lz4b200
