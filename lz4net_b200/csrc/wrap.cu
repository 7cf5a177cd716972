// wrap.cu -- kernels + launchers of the Wrap / Unwrap packet in device memory (see lz4_wrap.cuh for the rules).
#include "kernels.h"
#include "lz4_wrap.cuh"

namespace lz4b200 {

constexpr int PREP_THREADS = 256;
constexpr int FINISH_THREADS = 256;                    // 8 packets per CTA, a warp each
constexpr int FINISH_WARPS = FINISH_THREADS / 32;

static unsigned prep_grid(int32_t n) { return (unsigned)(((int64_t)n + PREP_THREADS - 1) / PREP_THREADS); }
static unsigned finish_grid(int32_t n) { return (unsigned)(((int64_t)n + FINISH_WARPS - 1) / FINISH_WARPS); }

__global__ void __launch_bounds__(PREP_THREADS)
lz4_wrap_prep_kernel(const int64_t* dst_off, const int32_t* src_len, const int32_t* dst_cap, int32_t n, WrapScratch w)
{
    const int64_t i = (int64_t)blockIdx.x * PREP_THREADS + threadIdx.x;
    if (i < n) wrap_prep_one(dst_off[i], src_len[i], dst_cap[i], w.off + i, w.len + i, w.cap + i);
}

__global__ void __launch_bounds__(FINISH_THREADS)
lz4_wrap_finish_kernel(const uint8_t* src, const int64_t* src_off, const int32_t* src_len, uint8_t* dst, const int64_t* dst_off,
                       const int32_t* dst_cap, int32_t* out_len, int32_t n, WrapScratch w)
{
    const int64_t i = (int64_t)blockIdx.x * FINISH_WARPS + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = (int)(threadIdx.x & 31);
    const int32_t len = src_len[i];
    const int32_t r = wrap_finish_one(src + src_off[i], len, dst_cap[i], w.res[i], dst + dst_off[i], lane);
    if (lane == 0) out_len[i] = r;
}

__global__ void __launch_bounds__(PREP_THREADS)
lz4_unwrap_prep_kernel(const uint8_t* src, const int64_t* src_off, const int32_t* src_len, const int32_t* dst_cap,
                       int32_t* out_len, int32_t n, WrapScratch w)
{
    const int64_t i = (int64_t)blockIdx.x * PREP_THREADS + threadIdx.x;
    if (i >= n) return;
    out_len[i] = unwrap_prep_one(src + src_off[i], src_len[i], dst_cap ? dst_cap[i] : 0x7FFFFFFF, w.len + i, w.cap + i);
    w.off[i] = src_off[i] + WRAP_HEADER;
}

__global__ void __launch_bounds__(FINISH_THREADS)
lz4_unwrap_finish_kernel(const uint8_t* src, const int64_t* src_off, uint8_t* dst, const int64_t* dst_off, int32_t* out_len,
                         int32_t n, WrapScratch w, const int* gate)
{
    if (gate && !*gate) return;
    const int64_t i = (int64_t)blockIdx.x * FINISH_WARPS + (threadIdx.x >> 5);
    if (i >= n) return;
    const int lane = (int)(threadIdx.x & 31);
    const int32_t r = unwrap_finish_one(src + src_off[i], out_len[i], w.len[i], w.cap[i], w.res[i], dst + dst_off[i], lane);
    simt::syncwarp(0xFFFFFFFFu);                        // (every lane has read out_len[i] before lane 0 replaces it)
    if (lane == 0) out_len[i] = r;
}

cudaError_t launch_wrap_prep(const BatchArgs& a, const WrapScratch& w, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    lz4_wrap_prep_kernel<<<prep_grid(a.n_blocks), PREP_THREADS, 0, stream>>>(a.dst_off, a.src_len, a.dst_cap, a.n_blocks, w);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_wrap_finish(const BatchArgs& a, const WrapScratch& w, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    lz4_wrap_finish_kernel<<<finish_grid(a.n_blocks), FINISH_THREADS, 0, stream>>>(a.src, a.src_off, a.src_len, a.dst, a.dst_off,
                                                                                   a.dst_cap, a.out_len, a.n_blocks, w);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_unwrap_prep(const BatchArgs& a, const WrapScratch& w, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    lz4_unwrap_prep_kernel<<<prep_grid(a.n_blocks), PREP_THREADS, 0, stream>>>(a.src, a.src_off, a.src_len, a.dst_cap, a.out_len,
                                                                                a.n_blocks, w);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_unwrap_finish(const BatchArgs& a, const WrapScratch& w, const int* gate, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    lz4_unwrap_finish_kernel<<<finish_grid(a.n_blocks), FINISH_THREADS, 0, stream>>>(a.src, a.src_off, a.dst, a.dst_off, a.out_len,
                                                                                      a.n_blocks, w, gate);
    if (launches) ++*launches;
    return cudaGetLastError();
}

}  // namespace lz4b200
