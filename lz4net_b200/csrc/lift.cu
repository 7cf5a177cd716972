// lift.cu -- the staging kernel of the asynchronous decode and Unwrap from device-written offsets (lz4_lift.cuh).
#include "kernels.h"
#include "lz4_lift.cuh"

#include <algorithm>

namespace lz4b200 {

// Grid-stride over the m entries, then over the stage's slot[m] / 16 units.  No thread reads what another writes.
__global__ void __launch_bounds__(256) lz4_lift_kernel(const uint8_t* src, int64_t src_cap, const int64_t* slot, const int64_t* span,
                                                        int32_t m, const int32_t* bound, int64_t* so, int32_t* sl, int32_t* dc,
                                                        uint8_t* io)
{
    const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = t0; i < m; i += stride) lift_entry((int32_t)i, src, src_cap, slot, span, m, bound, so, sl, dc);
    const int64_t units = slot[m] >> 4;
    for (int64_t u = t0; u < units; u += stride) lift_unit(u, src, src_cap, slot, span, m, bound, io);
}

__global__ void __launch_bounds__(256) lz4_lift_status_kernel(int64_t src_cap, const int64_t* span, int32_t m, const int32_t* bound,
                                                               int32_t* out)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) lift_status((int32_t)i, src_cap, span, m, bound, out);
}

cudaError_t launch_lift(const uint8_t* src, int64_t src_cap, const int64_t* slot, const int64_t* span, int32_t m, int64_t slot_bytes,
                        const int32_t* bound, int64_t* so, int32_t* sl, int32_t* dc, uint8_t* io, const DeviceInfo& dev,
                        cudaStream_t stream, int64_t* launches)
{
    if (m <= 0) return cudaSuccess;
    const int64_t work = std::max<int64_t>(m, slot_bytes >> 4);
    const int64_t blocks = std::min<int64_t>((work + 255) / 256, (int64_t)dev.num_sms * 16);
    lz4_lift_kernel<<<(unsigned)blocks, 256, 0, stream>>>(src, src_cap, slot, span, m, bound, so, sl, dc, io);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_lift_status(int64_t src_cap, const int64_t* span, int32_t m, const int32_t* bound, int32_t* out, cudaStream_t stream,
                               int64_t* launches)
{
    if (m <= 0) return cudaSuccess;
    lz4_lift_status_kernel<<<(unsigned)((m + 255) / 256), 256, 0, stream>>>(src_cap, span, m, bound, out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

}  // namespace lz4b200
