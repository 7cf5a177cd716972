// encode.cu -- kernels + launchers for the fast and the HC encoders.
#include "kernels.h"
#include "lz4_encode.cuh"
#include "lz4hc_encode.cuh"
#include "lz4hc_warp.cuh"
#include "lz4hc_window.cuh"

#include <algorithm>

namespace lz4b200 {

// ---- fast encoder: one warp per block, persistent, dynamic block hand-out --------------------------------------------
// All encoder warps of an SM live in ONE CTA (up to 14 warps x 16 KiB position tables = 224 KiB of dynamic shared
// memory -- separate CTAs would each pay 1 KiB of system-reserved shared memory, which costs the 14th warp).  The warps
// never synchronise with each other.  (The launch bound only tells ptxas how many registers it may use: 65536 / 448.)
// Tried and dropped: more warp-per-block encoders with their tables in an L2-resident global arena (the register cap
// spills the parse and a table round trip becomes an L2 round trip), and a 15th warp whose lanes each encode a block of
// their own with the table in global memory (its scattered table and candidate traffic costs the 14 warps more L2 hits
// than its own blocks add).  The same shared-memory budget holds on H100 (227 KiB per block, 228 KiB per SM).
constexpr int ENC_MAX_WARPS = 14;

template <int DUP>
__global__ void __launch_bounds__(32 * ENC_MAX_WARPS, 1)
lz4_encode_fast_kernel(BatchArgs a, uint32_t* counter, EncTune tune)
{
    extern __shared__ __align__(16) uint8_t smem[];
    EncShared* sh = (EncShared*)smem + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    for (;;) {
        uint32_t b = 0;
        if (lane == 0) b = atomicAdd(counter, 1u);
        b = simt::shfl(0xFFFFFFFFu, b, 0);
        if (b >= (uint32_t)a.n_blocks) break;
        const int r = encode_block<DUP, 0>(sh, a.src + a.src_off[b], a.src_len[b], a.dst + a.dst_off[b], a.dst_cap[b], lane, tune);
        if (lane == 0) a.out_len[b] = r;
    }
}

template <int DUP>
static cudaError_t launch_fast_t(const BatchArgs& a, uint32_t* counter, int dyn, long long grid, int warps, const EncTune& tune, cudaStream_t stream)
{
    cudaError_t e = cudaFuncSetAttribute(lz4_encode_fast_kernel<DUP>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn);
    if (e != cudaSuccess) return e;
    lz4_encode_fast_kernel<DUP><<<(unsigned)grid, 32 * warps, dyn, stream>>>(a, counter, tune);
    return cudaGetLastError();
}

cudaError_t launch_encode_fast(const BatchArgs& a, uint32_t* counter, int warps_per_sm, const int* tune4, int variant,
                               const DeviceInfo& dev, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    int max_warps = dev.smem_optin / (int)sizeof(EncShared);
    if (max_warps > ENC_MAX_WARPS) max_warps = ENC_MAX_WARPS;
    if (max_warps < 1) max_warps = 1;
    if (warps_per_sm < 1 || warps_per_sm > max_warps) warps_per_sm = max_warps;
    // small batches: spread the blocks over the SMs first
    long long grid = dev.num_sms;
    int warps = warps_per_sm;
    if (a.n_blocks < (long long)dev.num_sms * warps) {
        warps = (int)((a.n_blocks + dev.num_sms - 1) / dev.num_sms);
        grid = (a.n_blocks + warps - 1) / warps;
    }
    const int dyn = warps * (int)sizeof(EncShared);
    cudaError_t e = cudaMemsetAsync(counter, 0, sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    if (launches) ++*launches;
    EncTune tune; tune.pf_dist = tune4[0]; tune.lane_copy_max = tune4[1]; tune.probe_max = tune4[2]; tune.wide_min = tune4[3];
    // variant: how same-hash iterations of one round are found (lz4_encode.cuh): 1 = always exact (one vote per hash bit),
    // 2 = through the table, pairs resolved in place (default)
    return variant == 1 ? launch_fast_t<1>(a, counter, dyn, grid, warps, tune, stream)
                        : launch_fast_t<2>(a, counter, dyn, grid, warps, tune, stream);
}

// ---- HC encoder: one THREAD per block, state arena in global memory -------------------------------------------------
constexpr int HC_THREADS = 32;

__global__ void __launch_bounds__(HC_THREADS)
lz4_encode_hc_kernel(BatchArgs a, uint8_t* arena, uint32_t* counter)
{
    const size_t slot = (size_t)blockIdx.x * HC_THREADS + threadIdx.x;
    void* state = arena + slot * HC_STATE_BYTES;
    for (;;) {
        const uint32_t b = atomicAdd(counter, 1u);
        if (b >= (uint32_t)a.n_blocks) break;
        a.out_len[b] = hc_encode_block(state, a.src + a.src_off[b], a.src_len[b], a.dst + a.dst_off[b], a.dst_cap[b]);
    }
}

size_t hc_scratch_bytes(int concurrency)
{
    size_t slots = ((size_t)concurrency + HC_THREADS - 1) / HC_THREADS * HC_THREADS;
    return slots * HC_STATE_BYTES;
}

static cudaError_t launch_hc_threads(const BatchArgs& a, void* scratch, int concurrency, uint32_t* counter,
                                     cudaStream_t stream, int64_t* launches)
{
    long long ctas = ((long long)concurrency + HC_THREADS - 1) / HC_THREADS;
    long long want = ((long long)a.n_blocks + HC_THREADS - 1) / HC_THREADS;
    if (ctas > want) ctas = want;
    if (ctas < 1) ctas = 1;
    lz4_encode_hc_kernel<<<(unsigned)ctas, HC_THREADS, 0, stream>>>(a, (uint8_t*)scratch, counter);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_encode_hc(const BatchArgs& a, void* scratch, int concurrency, uint32_t* counter,
                             const DeviceInfo&, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    cudaError_t e = cudaMemsetAsync(counter, 0, sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    return launch_hc_threads(a, scratch, concurrency, counter, stream, launches);
}

// ---- HC encoder, blocks <= 64 KiB: one WARP per block on a static index (lz4hc_warp.cuh) -----------------------------
// One 32-thread CTA per warp.  SMEM variant: the block's bytes take 64 KiB of shared memory, so at most three CTAs share an
// SM (fewer are forced by asking for more shared memory than the CTA uses).  Global variant: no shared memory, up to 32
// CTAs per SM, the block read through L1 / L2.  Each CTA owns HCW_INDEX_BYTES of the scratch arena (rank / sorted tables).
// MINB = CTAs per SM the register budget is cut for (SMEM: 3; global variant: 16 -> <= 128 registers, 32 -> 64)
template <bool SMEM, int MINB>
__global__ void __launch_bounds__(32, MINB)
lz4_encode_hcw_kernel(BatchArgs a, uint8_t* arena, uint32_t* counter)
{
    extern __shared__ __align__(16) uint8_t smem[];
    const simt::smem_ref sm = simt::smem_ref_of(smem);
    void* index = arena + (size_t)blockIdx.x * HCW_INDEX_BYTES;
    const int lane = threadIdx.x;
    for (;;) {
        uint32_t b = 0;
        if (lane == 0) b = atomicAdd(counter, 1u);
        b = simt::shfl(0xFFFFFFFFu, b, 0);
        if (b >= (uint32_t)a.n_blocks) break;
        const int r = hcw_encode_block<SMEM>(sm, index, a.src + a.src_off[b], a.src_len[b], a.dst + a.dst_off[b], a.dst_cap[b], lane);
        if (lane == 0) a.out_len[b] = r;
        simt::syncwarp(0xFFFFFFFFu);                       // the next block reuses the shared memory and the index
    }
}

// the blocks the warp kernel handed back (larger than 64 KiB, or a state its static index does not describe): exact
// thread-per-block encoder, each thread looks at a stride of the batch
__global__ void __launch_bounds__(HC_THREADS)
lz4_encode_hc_marked_kernel(BatchArgs a, uint8_t* arena)
{
    const size_t slot = (size_t)blockIdx.x * HC_THREADS + threadIdx.x;
    void* state = arena + slot * HC_STATE_BYTES;
    const size_t stride = (size_t)gridDim.x * HC_THREADS;
    for (size_t b = slot; b < (size_t)a.n_blocks; b += stride)
        if (a.out_len[b] == HCW_FALLBACK)
            a.out_len[b] = hc_encode_block(state, a.src + a.src_off[b], a.src_len[b], a.dst + a.dst_off[b], a.dst_cap[b]);
}

constexpr int HCW_FALLBACK_THREADS = 4096;                 // thread-per-block slots kept for handed-back blocks (1 GiB of state)

// ---- HC encoder, blocks > 64 KiB: one WARP per block over a sliding 64 KiB window (lz4hc_window.cuh) --------------------
// Takes the blocks the warp kernel handed back for their size; whatever it hands back itself stays marked for the thread
// kernel.  One 32-thread CTA per warp, nothing in shared memory, HCWW_INDEX_BYTES of the arena per CTA.  HCWW_WARPS CTAs
// per SM: the launch bound lets ptxas use 128 registers, and it needs 120 without spilling or local memory (-Xptxas -v).
constexpr int HCWW_WARPS = 16;

__global__ void __launch_bounds__(32, HCWW_WARPS)
lz4_encode_hcw_window_kernel(BatchArgs a, uint8_t* arena, uint32_t* counter)
{
    void* index = arena + (size_t)blockIdx.x * HCWW_INDEX_BYTES;
    const int lane = threadIdx.x;
    for (;;) {
        uint32_t b = 0;
        if (lane == 0) b = atomicAdd(counter, 1u);
        b = simt::shfl(0xFFFFFFFFu, b, 0);
        if (b >= (uint32_t)a.n_blocks) break;
        if (a.out_len[b] != HCW_FALLBACK || a.src_len[b] <= HCW_MAX_BLOCK) continue;      // (the same values in every lane)
        const int r = hcww_encode_block(index, a.src + a.src_off[b], a.src_len[b], a.dst + a.dst_off[b], a.dst_cap[b], lane);
        if (lane == 0) a.out_len[b] = r;
        simt::syncwarp(0xFFFFFFFFu);                       // the next block reuses the index
    }
}

// CTAs of the window kernel: one per block above 64 KiB up to HCWW_WARPS per SM (n_large < 0: not known on the host, the
// batch's block count stands for it)
static int hcww_grid(int32_t n_blocks, int32_t n_large, const DeviceInfo& dev)
{
    long long g = (long long)dev.num_sms * HCWW_WARPS, want = n_large < 0 ? n_blocks : n_large;
    return (int)(g < want ? g : want);
}

static int hcw_warps(int variant, int warps_per_sm) { const int mx = variant == 1 ? 3 : 32; return warps_per_sm < 1 || warps_per_sm > mx ? mx : warps_per_sm; }

static int hcw_grid(int32_t n_blocks, int variant, int warps_per_sm, const DeviceInfo& dev)
{
    long long g = (long long)dev.num_sms * hcw_warps(variant, warps_per_sm);
    if (g > n_blocks) g = n_blocks;
    return g < 1 ? 1 : (int)g;
}

size_t hcw_scratch_bytes(int32_t n_blocks, int32_t n_large, int variant, int warps_per_sm, const DeviceInfo& dev)
{
    // the three kernels run one after the other on the same arena
    const size_t index = (size_t)hcw_grid(n_blocks, variant, warps_per_sm, dev) * HCW_INDEX_BYTES;
    const size_t window = (size_t)hcww_grid(n_blocks, n_large, dev) * HCWW_INDEX_BYTES;
    const size_t back = hc_scratch_bytes((int)(n_blocks < HCW_FALLBACK_THREADS ? (n_blocks < 1 ? 1 : n_blocks) : HCW_FALLBACK_THREADS));
    return std::max(index, std::max(window, back));
}

// variant 1: block staged in shared memory (<= 3 warps per SM); 2: nothing in shared memory (<= 32 warps per SM).
// Then the window kernel over the blocks above 64 KiB, then the thread kernel over whatever is still handed back.
// counter: four words, zero on entry (the warp kernel's ticket, the window kernel's).
static cudaError_t launch_hc_warps(const BatchArgs& a, void* scratch, int variant, int warps_per_sm, int32_t n_large, uint32_t* counter,
                                   const DeviceInfo& dev, cudaStream_t stream, int64_t* launches)
{
    const int warps = hcw_warps(variant, warps_per_sm);
    const int grid = hcw_grid(a.n_blocks, variant, warps_per_sm, dev);
    cudaError_t e = cudaSuccess;
    if (variant == 1) {
        // residency: the CTA needs HCW_SMEM_BYTES; asking for a larger share of the SM keeps the others out
        int dyn = HCW_SMEM_BYTES;
        if (warps < 3) { const int share = dev.smem_per_sm / warps - 2048; if (share > dyn) dyn = share < dev.smem_optin ? share : dev.smem_optin; }
        e = cudaFuncSetAttribute(lz4_encode_hcw_kernel<true, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn);
        if (e != cudaSuccess) return e;
        lz4_encode_hcw_kernel<true, 3><<<(unsigned)grid, 32, dyn, stream>>>(a, (uint8_t*)scratch, counter);
    } else {
        // Residency below 32 CTAs per SM is a matter of the grid alone: CTAs are placed breadth-first over the SMs and the
        // kernel is persistent.  No shared-memory carve-out preference: asking for "all L1" (cudaSharedmemCarveoutMaxL1)
        // left room for the system-reserved KiB of only a handful of CTAs per SM -- 16 to 32 warps per SM all ran at the
        // speed of 8 (tools/hc_ab.py: identical times); the default lets the driver size it for the occupancy.
        if (warps <= 16) lz4_encode_hcw_kernel<false, 16><<<(unsigned)grid, 32, 0, stream>>>(a, (uint8_t*)scratch, counter);
        else             lz4_encode_hcw_kernel<false, 32><<<(unsigned)grid, 32, 0, stream>>>(a, (uint8_t*)scratch, counter);
    }
    if (launches) ++*launches;
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (n_large != 0) {
        lz4_encode_hcw_window_kernel<<<(unsigned)hcww_grid(a.n_blocks, n_large, dev), 32, 0, stream>>>(a, (uint8_t*)scratch, counter + 1);
        if (launches) ++*launches;
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    const int back = a.n_blocks < HCW_FALLBACK_THREADS ? a.n_blocks : HCW_FALLBACK_THREADS;
    lz4_encode_hc_marked_kernel<<<(unsigned)((back + HC_THREADS - 1) / HC_THREADS), HC_THREADS, 0, stream>>>(a, (uint8_t*)scratch);
    if (launches) ++*launches;
    return cudaGetLastError();
}

cudaError_t launch_encode_hcw(const BatchArgs& a, void* scratch, int variant, int warps_per_sm, int32_t n_large, uint32_t* counter,
                              const DeviceInfo& dev, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    cudaError_t e = cudaMemsetAsync(counter, 0, 2 * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    return launch_hc_warps(a, scratch, variant, warps_per_sm, n_large, counter, dev, stream, launches);
}

// ---- HC, kernel chosen per batch -------------------------------------------------------------------------------------
// Small batches (at most three blocks per SM): the shared-memory warp kernel, whose time per block is the shortest by far
// (a lone thread of the thread kernel walks its block's chains one dependent load at a time); larger batches: the warp
// kernel with nothing in shared memory at 32 warps per SM.  Blocks above 64 KiB go to the window kernel either way: it
// was ahead of the thread kernel on every batch of such blocks timed (profiles/README.md).
static int hc_auto_variant(int32_t n_blocks, const DeviceInfo& dev) { return n_blocks <= 3 * dev.num_sms ? 1 : 2; }

size_t hc_auto_scratch_bytes(int32_t n_blocks, int32_t n_large, const DeviceInfo& dev)
{
    return hcw_scratch_bytes(n_blocks, n_large, hc_auto_variant(n_blocks, dev), 0, dev);
}

cudaError_t launch_encode_hc_auto(const BatchArgs& a, void* scratch, int32_t n_large, uint32_t* counter /* four words */,
                                  const DeviceInfo& dev, cudaStream_t stream, int64_t* launches)
{
    return launch_encode_hcw(a, scratch, hc_auto_variant(a.n_blocks, dev), 0, n_large, counter, dev, stream, launches);
}

}  // namespace lz4b200
