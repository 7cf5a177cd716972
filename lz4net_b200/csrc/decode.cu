// decode.cu -- kernel + launcher for the batched decoder (see lz4_decode.cuh for the algorithm).
#include "kernels.h"
#include "lz4_decode.cuh"
#include "lz4_decode_lpb.cuh"
#include "lz4_measure.cuh"
#include "lz4_packed.cuh"

namespace lz4b200 {

int decode_lanes_for_ratio(double ratio);        // (host + device: below)
__host__ __device__ int decode_lanes_for_ratio(double ratio) { return ratio > 0.95 ? 32 : (ratio < 0.05 ? 16 : (ratio < 0.45 ? 104 : 108)); }

constexpr int DEC_THREADS = 128;
// registers: a cap of 40 (12 CTAs/SM) spills the loop state of the sub-warp variants to local memory (measured:
// 2 LDL per sequence, half of them L1 misses) -- leave the compiler its ~56 registers, 9 CTAs = 36 warps per SM.
constexpr int DEC_MIN_CTAS = 9;

// Persistent CTAs; each group of G lanes pulls the next block index from a global counter.
// (the staged sub-warp variants are limited to 8 CTAs per SM by shared memory anyway: let them have 64 registers)
template <int G, bool KNOWN, bool STAGED>
__global__ void __launch_bounds__(DEC_THREADS, (STAGED && G < 32) ? 8 : DEC_MIN_CTAS)
lz4_decode_kernel(BatchArgs a, uint32_t* counter, const int* pick, int code)
{
    // auto-selected launches: every candidate kernel is enqueued, the one the pick kernel chose runs, the others leave at once
    if (pick && *pick != code) return;
    constexpr int GROUPS = DEC_THREADS / G;
    __shared__ DecRing<G> rings[GROUPS];
    __shared__ DecStage<G> stages[STAGED ? GROUPS : 1];
    const int grp = threadIdx.x / G;
    const int wl = threadIdx.x & 31;                               // lane within the warp
    const int leader = wl & ~(G - 1);
    const uint32_t gmask = (G == 32) ? 0xFFFFFFFFu : (((1u << G) - 1u) << leader);

    DecStream<G> st;
    st.ring = &rings[grp]; st.lane = wl - leader; st.gmask = gmask;
    st.gbase = 0;
    if (st.lane == 0) {
        for (int s = 0; s < DEC_SLOTS; s++) simt::mbar_init(&st.ring->bar[s], 1);
        simt::fence_mbar_init();
    }
    simt::syncwarp(gmask);

    for (;;) {
        uint32_t b = 0;
        if (st.lane == 0) b = atomicAdd(counter, 1u);
        b = simt::shfl(gmask, b, leader);
        if (b >= (uint32_t)a.n_blocks) break;
        const int r = STAGED
            ? decode_block_staged<G, KNOWN>(st, &stages[STAGED ? grp : 0], a.src + a.src_off[b], a.src_len[b], a.dst + a.dst_off[b], a.dst_cap[b])
            : decode_block<G, KNOWN>(st, a.src + a.src_off[b], a.src_len[b], a.dst + a.dst_off[b], a.dst_cap[b]);
        if (st.lane == 0) a.out_len[b] = r;
    }
}

// Decoder choice for a device-memory batch, made ON the device (the call stays asynchronous): compressed / raw bytes over
// the first blocks of the batch -> the same rule as lanes_for_ratio() on the host (capi.cu, tools/sweep.py): incompressible
// data is long literal runs (whole warps, 128-bit copies), nearly-empty streams are long matches, everything between is
// sequence-dense (the denser, the smaller the group; both output-staged).
// gate (may be null): a device flag; 0 makes the pick 0, which no decoder kernel answers to (the packed decode when its
// output does not fit).  fixed != 0: the code of the one kernel a pinned decode_lanes setting launched.
__global__ void __launch_bounds__(256) lz4_decode_pick_kernel(const int32_t* src_len, const int32_t* dst_cap, int32_t n, int* pick,
                                                              const int* gate, int fixed)
{
    __shared__ unsigned long long sc[8], sr[8];
    unsigned long long c = 0, r = 0;
    const int m = n < 8192 ? n : 8192;
    for (int i = threadIdx.x; i < m; i += 256) { c += (unsigned)(src_len[i] > 0 ? src_len[i] : 0); r += (unsigned)(dst_cap[i] > 0 ? dst_cap[i] : 0); }
    for (int d = 16; d > 0; d >>= 1) { c += __shfl_down_sync(0xFFFFFFFFu, c, d); r += __shfl_down_sync(0xFFFFFFFFu, r, d); }
    if ((threadIdx.x & 31) == 0) { sc[threadIdx.x >> 5] = c; sr[threadIdx.x >> 5] = r; }
    __syncthreads();
    if (threadIdx.x == 0) {
        c = r = 0;
        for (int i = 0; i < 8; i++) { c += sc[i]; r += sr[i]; }
        const double ratio = r ? (double)c / (double)r : 1.0;
        *pick = gate && !*gate ? 0 : (fixed ? fixed : decode_lanes_for_ratio(ratio));
    }
}

template <int G, bool KNOWN, bool STAGED>
static cudaError_t launch_one(const BatchArgs& a, uint32_t* counter, const DeviceInfo& dev, cudaStream_t stream, const int* pick, int code)
{
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lz4_decode_kernel<G, KNOWN, STAGED>, DEC_THREADS, 0);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) per_sm = 1;
    constexpr int GROUPS = DEC_THREADS / G;
    long long want = ((long long)a.n_blocks + GROUPS - 1) / GROUPS;
    long long grid = (long long)dev.num_sms * per_sm;
    if (grid > want) grid = want;
    if (grid < 1) grid = 1;
    lz4_decode_kernel<G, KNOWN, STAGED><<<(unsigned)grid, DEC_THREADS, 0, stream>>>(a, counter, pick, code);
    return cudaGetLastError();
}

template <int G>
static cudaError_t launch_g(const BatchArgs& a, bool known, bool staged, uint32_t* counter, const DeviceInfo& dev, cudaStream_t stream,
                            const int* pick, int code)
{
    if (staged) return known ? launch_one<G, true, true>(a, counter, dev, stream, pick, code) : launch_one<G, false, true>(a, counter, dev, stream, pick, code);
    return known ? launch_one<G, true, false>(a, counter, dev, stream, pick, code) : launch_one<G, false, false>(a, counter, dev, stream, pick, code);
}

// ---- lane-per-block decoder (lz4_decode_lpb.cuh): one CTA per SM, as many warps as shared memory holds rings for --------
// Geometry (tools/sweep.py): 128-byte input ring, 256-byte output window, runs up to 32 bytes copied by the lane,
// requests waited for at the top of the next iteration, two sequences per iteration: 16 warps = 512 blocks in flight per SM.
// (256 / 512-byte rings with 64-byte runs and one-iteration-ahead requests -- 8 warps -- were slower on E50 and ETEXT alike:
// this kernel lives on resident warps.)
typedef LpbGeom<128, 256, 32, 0, 2> LpbDefault;
// Warps per CTA: what 227 KiB of shared memory hold rings for, rounded DOWN to a multiple of four -- ptxas budgets registers
// for the block size rounded up to 128 threads (17 warps were given the 96 registers of 20 and spilled the copy loops).
template <class GEO> constexpr int lpb_warps() { return (int)((232448 / sizeof(LpbShared<GEO>)) / 4 * 4) > 0 ? (int)((232448 / sizeof(LpbShared<GEO>)) / 4 * 4) : 1; }

template <bool KNOWN, class GEO>
__global__ void __launch_bounds__(32 * lpb_warps<GEO>(), 1)
lz4_decode_lpb_kernel(BatchArgs a, uint32_t* counter, const int* pick, int takes108)
{
    // auto-selected launches: the dense class (104) is this kernel's, the middle class (108) when the batch fills its waves
    if (pick && *pick != 104 && !(takes108 && *pick == 108)) return;
    extern __shared__ __align__(128) uint8_t lpb_smem[];
    LpbShared<GEO>* sh = (LpbShared<GEO>*)lpb_smem + (threadIdx.x >> 5);
    const LpbBatch b{a.src, a.src_off, a.src_len, a.dst, a.dst_off, a.dst_cap, a.out_len, a.n_blocks};
    lpb_decode_warp<KNOWN, GEO>(sh, b, counter, (int)(threadIdx.x & 31));
}

// The lane-per-block decoder holds one block per lane (on H100 132 x 16 x 32 = 67 584 at a time) and blocks of one class take
// about equally long, so a batch is worked off in waves: below half a wave the group kernels are ahead; on token-dense
// data (class 104) it is 1.4-1.6x the 4-lane group kernel and pays from there on; on the middle class (108) its edge over
// the 8-lane kernel is ~11 %, which a last wave that is less than ~90 % full gives back.
static bool lpb_pays(int64_t n_blocks, const DeviceInfo& dev, bool middle_class)
{
    const int64_t wave = (int64_t)dev.num_sms * 32 * lpb_warps<LpbDefault>();
    if (n_blocks * 2 < wave) return false;
    if (!middle_class) return true;
    const int64_t waves = (n_blocks + wave - 1) / wave;
    return n_blocks * 10 >= waves * wave * 9;
}

template <bool KNOWN, class GEO>
static cudaError_t launch_lpb(const BatchArgs& a, uint32_t* counter, const DeviceInfo& dev, cudaStream_t stream, const int* pick, int takes108)
{
    int warps = dev.smem_optin / (int)sizeof(LpbShared<GEO>);
    if (warps > lpb_warps<GEO>()) warps = lpb_warps<GEO>();
    if (warps < 1) return cudaErrorInvalidConfiguration;
    long long grid = dev.num_sms;
    const long long want_warps = ((long long)a.n_blocks + 31) / 32;          // one block per lane
    if (want_warps < grid * warps) {                                         // small batch: spread the warps over the SMs first
        warps = (int)((want_warps + grid - 1) / grid);
        grid = (want_warps + warps - 1) / warps;
    }
    const int dyn = warps * (int)sizeof(LpbShared<GEO>);
    cudaError_t e = cudaFuncSetAttribute(lz4_decode_lpb_kernel<KNOWN, GEO>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn);
    if (e != cudaSuccess) return e;
    lz4_decode_lpb_kernel<KNOWN, GEO><<<(unsigned)grid, 32 * warps, dyn, stream>>>(a, counter, pick, takes108);
    return cudaGetLastError();
}

cudaError_t launch_decode(const BatchArgs& a, bool known_len, int lanes, uint32_t* counter,
                          const DeviceInfo& dev, cudaStream_t stream, int64_t* launches, const int* gate)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    cudaError_t e = cudaMemsetAsync(counter, 0, 4 * sizeof(uint32_t), stream);     // [block counter, decoder pick, two more block counters]
    if (e != cudaSuccess) return e;
    if (launches) ++*launches;
    int* pick = (int*)(counter + 1);                 // (the context hands out counters in fours: [block counter, pick, two more counters])
    if (lanes != 0) {
        // a pinned decoder.  Behind a gate the pick kernel goes first and passes the gate on as that kernel's code (or 0);
        // without one the kernel gets no pick, and then ignores code and takes108.
        const int code = lanes == 1 ? 104 : lanes;
        if (gate) {
            lz4_decode_pick_kernel<<<1, 256, 0, stream>>>(a.src_len, a.dst_cap, a.n_blocks, pick, gate, code);
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
            if (launches) ++*launches;
        } else {
            pick = nullptr;
        }
        const bool staged = lanes >= 100;            // lanes = 100 + G selects the output-staged variant
        switch (lanes % 100) {
        case 1:  return known_len ? launch_lpb<true, LpbDefault>(a, counter, dev, stream, pick, 0) : launch_lpb<false, LpbDefault>(a, counter, dev, stream, pick, 0);
        case 4:  return launch_g<4>(a, known_len, staged, counter, dev, stream, pick, code);
        case 8:  return launch_g<8>(a, known_len, staged, counter, dev, stream, pick, code);
        case 16: return launch_g<16>(a, known_len, staged, counter, dev, stream, pick, code);
        default: return launch_g<32>(a, known_len, staged, counter, dev, stream, pick, code);
        }
    }
    // auto: pick on the device, enqueue the four candidates (three of them return at once)
    lz4_decode_pick_kernel<<<1, 256, 0, stream>>>(a.src_len, a.dst_cap, a.n_blocks, pick, gate, 0);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    if (launches) *launches += 2;
    if ((e = launch_g<32>(a, known_len, false, counter, dev, stream, pick, 32)) != cudaSuccess) return e;
    if ((e = launch_g<16>(a, known_len, false, counter, dev, stream, pick, 16)) != cudaSuccess) return e;
    // Sequence-dense classes.  The lane-per-block decoder works a batch off in waves of one block per lane; it gets the
    // whole waves, the group kernels the rest (a last wave that is 46 % full, as in a 262 144-block batch, costs the
    // token-dense class a quarter of its rate).  Batches below one wave: lpb_pays().
    const int64_t wave = (int64_t)dev.num_sms * 32 * lpb_warps<LpbDefault>();
    const int64_t head = a.n_blocks >= wave ? a.n_blocks / wave * wave : (lpb_pays(a.n_blocks, dev, false) ? a.n_blocks : 0);
    const bool head108 = a.n_blocks >= wave || lpb_pays(a.n_blocks, dev, true);
    if (head > 0) {
        BatchArgs h = a; h.n_blocks = (int32_t)head;
        if (launches) ++*launches;
        e = known_len ? launch_lpb<true, LpbDefault>(h, counter, dev, stream, pick, head108 ? 1 : 0) : launch_lpb<false, LpbDefault>(h, counter, dev, stream, pick, head108 ? 1 : 0);
        if (e != cudaSuccess) return e;
    }
    // the rest of the batch (or all of it) for the group kernels; class 108 also takes the head when the lanes did not
    uint32_t* tc = counter + 2;
    const int64_t skip104 = head, skip108 = head108 ? head : 0;
    auto tail = [&](int64_t skip) { BatchArgs r = a; r.src_off += skip; r.src_len += skip; r.dst_off += skip; r.dst_cap += skip; r.out_len += skip; r.n_blocks = (int32_t)(a.n_blocks - skip); return r; };
    if (a.n_blocks - skip108 > 0) { if (launches) ++*launches; if ((e = launch_g<8>(tail(skip108), known_len, true, tc, dev, stream, pick, 108)) != cudaSuccess) return e; }
    if (a.n_blocks - skip104 > 0) { if (launches) ++*launches; if ((e = launch_g<4>(tail(skip104), known_len, true, tc + 1, dev, stream, pick, 104)) != cudaSuccess) return e; }
    return cudaSuccess;
}

// ---- measure pass (lz4_measure.cuh): one thread per block, no shared memory ---------------------------------------------
constexpr int MEASURE_THREADS = 128;

template <bool KNOWN>
__global__ void __launch_bounds__(MEASURE_THREADS)
lz4_measure_kernel(BatchArgs a)
{
    const int64_t i = (int64_t)blockIdx.x * MEASURE_THREADS + threadIdx.x;
    if (i >= a.n_blocks) return;
    const int cap = a.dst_cap ? a.dst_cap[i] : 0x7FFFFFFF;          // no capacities: INT32_MAX for every block
    a.out_len[i] = measure_block<KNOWN>(a.src + a.src_off[i], a.src_len[i], cap);
}

cudaError_t launch_measure(const BatchArgs& a, bool known_len, const DeviceInfo&, cudaStream_t stream, int64_t* launches)
{
    if (a.n_blocks <= 0) return cudaSuccess;
    const unsigned grid = (unsigned)(((int64_t)a.n_blocks + MEASURE_THREADS - 1) / MEASURE_THREADS);
    if (known_len) lz4_measure_kernel<true><<<grid, MEASURE_THREADS, 0, stream>>>(a);
    else           lz4_measure_kernel<false><<<grid, MEASURE_THREADS, 0, stream>>>(a);
    if (launches) ++*launches;
    return cudaGetLastError();
}

// Between the scan and the decode of the packed decodes (lz4_packed.cuh): capacities, the "fits" gate and, for a stage of
// the host pipeline, the blocks' absolute offsets behind the running total of the earlier stages.  base_in and total_out
// are different cells: every thread reads the one, thread 0 writes the other.
__global__ void __launch_bounds__(256) lz4_packed_prep_kernel(const int32_t* size, const int64_t* out_off, int32_t n,
                                                              int64_t total_cap, int32_t* cap, int* fits,
                                                              const int64_t* base_in, int64_t* abs_off, int64_t* total_out)
{
    packed_place((int64_t)blockIdx.x * 256 + threadIdx.x, size, out_off, n, base_in ? *base_in : 0, total_cap, cap, abs_off, fits,
                 total_out);
}

cudaError_t launch_packed_prep(const int32_t* size, const int64_t* out_off, int32_t n, int64_t total_cap, int32_t* cap, int* fits,
                               cudaStream_t stream, int64_t* launches, const int64_t* base_in, int64_t* abs_off, int64_t* total_out)
{
    if (n <= 0) return cudaSuccess;
    lz4_packed_prep_kernel<<<(unsigned)(((int64_t)n + 255) / 256), 256, 0, stream>>>(size, out_off, n, total_cap, cap, fits,
                                                                                     base_in, abs_off, total_out);
    if (launches) ++*launches;
    return cudaGetLastError();
}

}  // namespace lz4b200
