// enc_phases.cu -- the fast encoder with its phase counters compiled in (enc_prof.cuh), for tools/enc_phases.py.
// Built by that script into a temporary directory with -DLZ4B200_ENC_PROF (or without it, to time the same harness
// uninstrumented).  The kernel is lz4_encode_fast_kernel<2> of encode.cu with the library's default tuning.
#include "lz4_encode.cuh"
#include <cuda_runtime.h>

using namespace lz4b200;

namespace {
constexpr int WARPS = 14;

__global__ void __launch_bounds__(32 * WARPS, 1)
enc_phases_kernel(const uint8_t* src, int bsize, int nblocks, uint8_t* dst, int cap, int* out_len, uint32_t* counter, EncTune tune)
{
    extern __shared__ __align__(16) uint8_t smem[];
    EncShared* sh = (EncShared*)smem + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    for (;;) {
        uint32_t b = 0;
        if (lane == 0) b = atomicAdd(counter, 1u);
        b = simt::shfl(0xFFFFFFFFu, b, 0);
        if (b >= (uint32_t)nblocks) break;
        const int r = encode_block<2, 0>(sh, src + (size_t)b * bsize, bsize, dst + (size_t)b * cap, cap, lane, tune);
        if (lane == 0) out_len[b] = r;
    }
}
}  // namespace

// Encodes nblocks blocks of bsize bytes `reps` times; returns 0 or a CUDA error code.  rows: EP_N counters summed over
// all warps and all repetitions (all zero in an uninstrumented build); ms: kernel time per repetition, CUDA events.
extern "C" int enc_phases_run(const uint8_t* h_src, int bsize, int nblocks, int reps, int* h_out_len,
                              unsigned long long* rows, float* ms)
{
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const int cap = bsize + bsize / 255 + 16, nwarps = sms * WARPS, dyn = WARPS * (int)sizeof(EncShared);
    const size_t nsrc = (size_t)nblocks * bsize, ndst = (size_t)nblocks * cap, nrow = (size_t)nwarps * EP_N;
    uint8_t *src = nullptr, *dst = nullptr; int* out_len = nullptr; uint32_t* counter = nullptr; unsigned long long* prof = nullptr;
    cudaMalloc(&src, nsrc); cudaMalloc(&dst, ndst); cudaMalloc(&out_len, nblocks * sizeof(int));
    cudaMalloc(&counter, sizeof(uint32_t)); cudaMalloc(&prof, nrow * sizeof(unsigned long long));
    cudaMemcpy(src, h_src, nsrc, cudaMemcpyHostToDevice);
    cudaMemset(prof, 0, nrow * sizeof(unsigned long long));
#if defined(LZ4B200_ENC_PROF)
    cudaMemcpyToSymbol(enc_prof_rows, &prof, sizeof(prof));
#endif
    cudaFuncSetAttribute(enc_phases_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn);
    EncTune tune; tune.pf_dist = 512;                              // the library's defaults (capi.cu)
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float total = 0.f;
    for (int r = 0; r < reps; r++) {
        cudaMemset(counter, 0, sizeof(uint32_t));
        cudaEventRecord(e0);
        enc_phases_kernel<<<sms, 32 * WARPS, dyn>>>(src, bsize, nblocks, dst, cap, out_len, counter, tune);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float t = 0.f; cudaEventElapsedTime(&t, e0, e1); total += t;
    }
    *ms = total / (reps > 0 ? reps : 1);
    cudaMemcpy(h_out_len, out_len, nblocks * sizeof(int), cudaMemcpyDeviceToHost);
    unsigned long long* h = new unsigned long long[nrow];
    cudaMemcpy(h, prof, nrow * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
    for (int k = 0; k < EP_N; k++) rows[k] = 0;
    for (size_t w = 0; w < (size_t)nwarps; w++) for (int k = 0; k < EP_N; k++) rows[k] += h[w * EP_N + k];
    delete[] h;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaFree(src); cudaFree(dst); cudaFree(out_len); cudaFree(counter); cudaFree(prof);
    return (int)cudaGetLastError();
}
