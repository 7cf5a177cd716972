// ubench.cu -- single-warp latency probes for the primitives the encoder's parse chain is built from (H100, sm_90a).
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench tools/ubench.cu ; run on an H100.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint64_t clk() { uint64_t c; asm volatile("mov.u64 %0, %%clock64;" : "=l"(c)); return c; }

template <int MODE>
__global__ void probe(uint32_t* out, uint64_t* cycles, const uint32_t* gmem, uint32_t seed)
{
    __shared__ uint32_t sm[8192];
    const uint32_t lane = threadIdx.x;
    for (int i = lane; i < 8192; i += 32) sm[i] = (i * 2654435761u) >> 19;
    __syncwarp();
    uint32_t x = seed + lane * 977u;
    constexpr int N = 256;
    uint64_t t0 = clk();
#pragma unroll 1
    for (int i = 0; i < N; i++) {
        if (MODE == 0) x = __match_any_sync(0xffffffffu, x * 2654435761u >> 19) + x;                 // distinct keys (mostly)
        if (MODE == 1) x = __match_any_sync(0xffffffffu, (x >> 20) & 1) + x;                          // two groups
        if (MODE == 2) x = __shfl_sync(0xffffffffu, x, (x >> 3) & 31) + 1;
        if (MODE == 3) x = __ballot_sync(0xffffffffu, x & 1) + x + 1;
        if (MODE == 4) x = sm[x & 8191] + 1 + x;                                                       // LDS chain
        if (MODE == 5) x = gmem[(x * 2654435761u >> 19) & 8191] + x;                                  // L1-resident 32 KB
        if (MODE == 6) x = gmem[(x * 2654435761u >> 8) & ((1u << 22) - 1)] + x;                      // 16 MB: L2-resident
        if (MODE == 7) {                                                                               // 13 ballots + select
            uint32_t h = x * 2654435761u >> 19, m = 0xffffffffu;
#pragma unroll
            for (int b = 0; b < 13; b++) { uint32_t v = __ballot_sync(0xffffffffu, (h >> b) & 1); m &= ((h >> b) & 1) ? v : ~v; }
            x += m;
        }
        if (MODE == 8) x = __reduce_add_sync(0xffffffffu, x) + lane;
        if (MODE == 9) { sm[x & 8191] = x; __syncwarp(); x = sm[(x + 1) & 8191] + x; }                 // STS -> LDS
    }
    uint64_t t1 = clk();
    out[lane] = x;
    if (lane == 0) cycles[0] = (t1 - t0) / N;
}

int main()
{
    uint32_t *out, *g; uint64_t* cyc;
    cudaMalloc(&out, 128); cudaMalloc(&cyc, 8); cudaMalloc(&g, 16 << 20);
    cudaMemset(g, 1, 16 << 20);
    const char* names[] = {"match_any distinct", "match_any 2 groups", "shfl", "ballot", "LDS chain", "LDG L1-hit chain",
                           "LDG L2-hit chain (16 MB)", "13 ballots + select", "redux add", "STS+sync+LDS"};
    for (int m = 0; m < 10; m++) {
        for (int rep = 0; rep < 2; rep++) {
            switch (m) {
            case 0: probe<0><<<1, 32>>>(out, cyc, g, 12345); break; case 1: probe<1><<<1, 32>>>(out, cyc, g, 12345); break;
            case 2: probe<2><<<1, 32>>>(out, cyc, g, 12345); break; case 3: probe<3><<<1, 32>>>(out, cyc, g, 12345); break;
            case 4: probe<4><<<1, 32>>>(out, cyc, g, 12345); break; case 5: probe<5><<<1, 32>>>(out, cyc, g, 12345); break;
            case 6: probe<6><<<1, 32>>>(out, cyc, g, 12345); break; case 7: probe<7><<<1, 32>>>(out, cyc, g, 12345); break;
            case 8: probe<8><<<1, 32>>>(out, cyc, g, 12345); break; case 9: probe<9><<<1, 32>>>(out, cyc, g, 12345); break;
            }
            cudaDeviceSynchronize();
        }
        uint64_t c; cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
        printf("%-28s %6llu cycles/iter (dependent chain, incl. ~6 ALU)\n", names[m], (unsigned long long)c);
    }
    printf("err=%s\n", cudaGetErrorString(cudaGetLastError()));
    return 0;
}
