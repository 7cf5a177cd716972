// land.cu -- the landing kernel of the asynchronous packed encode into page-locked host memory (lz4_land.cuh).
#include "kernels.h"
#include "lz4_land.cuh"

#include <algorithm>

namespace lz4b200 {

// Grid-stride over the m + 1 result entries, then over the stage's 16-byte units.  The stage's total is known only here:
// the launch is sized for the slots' bytes, the most it can be.  base_in and total_out are different cells: every thread reads
// the one, one thread writes the other.
__global__ void __launch_bounds__(256) lz4_land_kernel(const uint8_t* dense, const int64_t* dof, const int32_t* len,
                                                        const int64_t* off, int32_t m, const int64_t* base_in,
                                                        int64_t total_cap, uint8_t* dst, int64_t* out_off, int32_t* out_len,
                                                        int64_t* total_out)
{
    const int64_t base = base_in ? *base_in : 0;
    const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = t0; i <= m; i += stride) land_place(i, len, off, m, base, out_off, out_len, total_out);
    const int64_t total = off[m];
    if (base + total > total_cap) return;
    uint8_t* at = dst + base;
    const int64_t units = land_units(at, total);
    for (int64_t u = t0; u < units; u += stride) land_unit(u, dense, dof, off, m, at);
}

cudaError_t launch_land(const uint8_t* dense, const int64_t* dof, const int32_t* len, const int64_t* off, int32_t m,
                        int64_t dense_bytes, const int64_t* base_in, int64_t total_cap, uint8_t* dst, int64_t* out_off,
                        int32_t* out_len, int64_t* total_out, const DeviceInfo& dev, cudaStream_t stream, int64_t* launches)
{
    if (m <= 0) return cudaSuccess;
    const int64_t work = std::max<int64_t>((int64_t)m + 1, (dense_bytes >> 4) + 2);
    const int64_t blocks = std::min<int64_t>((work + 255) / 256, (int64_t)dev.num_sms * 16);
    lz4_land_kernel<<<(unsigned)blocks, 256, 0, stream>>>(dense, dof, len, off, m, base_in, total_cap, dst, out_off, out_len,
                                                          total_out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

}  // namespace lz4b200
