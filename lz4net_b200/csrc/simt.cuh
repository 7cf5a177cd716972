// simt.cuh -- the handful of warp / memory primitives the codec kernels are written against.
//
// Device build (nvcc, sm_90a): thin wrappers over the hardware instructions (SHFL / VOTE / MATCH, LDG/STG with
// cache hints, cp.async.bulk + mbarrier for TMA-style staging -> SASS UBLKCP / SYNCS).
// Test build (-DLZ4B200_SIMT_EMU, g++): the same names come from tests/simt_emu/simt_emu.h, a coroutine emulation
// of one warp used only by the CPU-side logic tests.  The product library is never built that way.
#pragma once
#include <stdint.h>

#if defined(LZ4B200_SIMT_EMU)
#include "simt_emu.h"
#else

#include <cuda_runtime.h>
#define SIMT_DEV __device__ __forceinline__
#define SIMT_MEM __device__ __forceinline__
#define SIMT_NOINLINE __device__ __noinline__

namespace simt {

SIMT_DEV uint32_t shfl(uint32_t mask, uint32_t v, int src) { return __shfl_sync(mask, v, src); }
SIMT_DEV uint32_t ballot(uint32_t mask, bool p) { return __ballot_sync(mask, p); }
SIMT_DEV uint32_t match_any(uint32_t mask, uint32_t v) { return __match_any_sync(mask, v); }
SIMT_DEV uint32_t reduce_max(uint32_t mask, uint32_t v) { return __reduce_max_sync(mask, v); }     // REDUX
SIMT_DEV void syncwarp(uint32_t mask) { __syncwarp(mask); }
SIMT_DEV int ffs(uint32_t v) { return __ffs((int)v); }
SIMT_DEV int clz(uint32_t v) { return __clz((int)v); }
SIMT_DEV int popc(uint32_t v) { return __popc(v); }
SIMT_DEV uint32_t funnel_r(uint32_t lo, uint32_t hi, uint32_t sh) { return __funnelshift_r(lo, hi, sh); }
SIMT_DEV uint32_t funnel_l(uint32_t lo, uint32_t hi, uint32_t sh) { return __funnelshift_l(lo, hi, sh); }     // high word of (hi:lo) << sh

// Opaque identity: stops the compiler from re-deriving a value from its parts at every use (e.g. a 64-bit pointer
// that it would otherwise rebuild from base + offset + lane on each store).
template <class T> SIMT_DEV T* keep(T* p) { asm volatile("" : "+l"(p)); return p; }
SIMT_DEV uint32_t keep(uint32_t v) { asm volatile("" : "+r"(v)); return v; }

// coherent loads (data this kernel wrote earlier: decoder back-references): plain ld.global, L1-cacheable.  They are
// always separated from the producing store of another lane by a __syncwarp(), which is a memory barrier for the
// compiler as well, so no asm/volatile is needed (and plain loads can be predicated instead of branched around).
SIMT_DEV uint8_t  ldg_u8(const uint8_t* p) { return *p; }
SIMT_DEV uint32_t ldg_u32(const void* p) { return *(const uint32_t*)p; }
SIMT_DEV uint4    ldg_v4(const void* p) { return *(const uint4*)p; }
// read-only path (kernel inputs)
SIMT_DEV uint8_t  ldg_nc_u8(const uint8_t* p) { return __ldg(p); }
SIMT_DEV uint32_t ldg_nc_u32(const void* p) { return __ldg((const uint32_t*)p); }
SIMT_DEV uint4    ldg_nc_v4(const void* p) { return __ldg((const uint4*)p); }
SIMT_DEV uint32_t ldg_u16(const uint16_t* p) { return *p; }
SIMT_DEV void stg_u8(uint8_t* p, uint8_t v) { *p = v; }
SIMT_DEV void stg_u16(uint16_t* p, uint32_t v) { *p = (uint16_t)v; }
SIMT_DEV void stg_u32(void* p, uint32_t v) { *(uint32_t*)p = v; }
SIMT_DEV void stg_v4(void* p, uint4 v) { *(uint4*)p = v; }
// L2 residency hints (no extra instruction: the policy travels in the access descriptor).  keep = evict-last, for input
// that will be probed again at random positions while its block is being parsed; stream = evict-first, for output that is
// written once and not read back.  (Measured and dropped: `ld.global.cg` probes, -20 %; `L1::no_allocate` probes lose the
// line in L2 as well, 30x DRAM read amplification.)
SIMT_DEV uint64_t l2_policy_keep() { uint64_t p; asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
SIMT_DEV uint64_t l2_policy_stream() { uint64_t p; asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
SIMT_DEV uint32_t ldg_nc_hint_u32(const void* p, uint64_t pol) { uint32_t v; asm("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol)); return v; }
SIMT_DEV void stg_hint_u8(uint8_t* p, uint32_t v, uint64_t pol) { asm volatile("st.global.L2::cache_hint.u8 [%0], %1, %2;" :: "l"(p), "r"(v), "l"(pol) : "memory"); }
// Scheduling fence without an instruction: `x` formally depends on `dep`, so the first use of x (the point where the
// warp waits for the load that produces it) cannot be scheduled before dep has been computed.
SIMT_DEV void tie(uint32_t& x, uint32_t dep) { asm volatile("" : "+r"(x) : "r"(dep)); }

// A block of shared memory addressed by its 32-bit shared-window address (one register, computed once; LDS/STS take
// it with an immediate-free register offset -- no generic-pointer conversion in the loop).
struct smem_ref { uint32_t a; };
SIMT_DEV smem_ref smem_ref_of(const void* p) { smem_ref r; r.a = (uint32_t)__cvta_generic_to_shared(p); asm volatile("" : "+r"(r.a)); return r; }
SIMT_DEV uint32_t lds_u16(smem_ref r, uint32_t off) { uint16_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(r.a + off) : "memory"); return v; }
SIMT_DEV uint32_t lds_u32(smem_ref r, uint32_t off) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(r.a + off) : "memory"); return v; }
SIMT_DEV uint32_t lds_u8(smem_ref r, uint32_t off) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(r.a + off) : "memory"); return v; }
SIMT_DEV uint4 lds_v4(smem_ref r, uint32_t off) { uint4 v; asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(r.a + off) : "memory"); return v; }
SIMT_DEV void sts_u8(smem_ref r, uint32_t off, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(r.a + off), "r"(v) : "memory"); }
SIMT_DEV void sts_u16(smem_ref r, uint32_t off, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" :: "r"(r.a + off), "h"((uint16_t)v) : "memory"); }
SIMT_DEV void sts_u32(smem_ref r, uint32_t off, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(r.a + off), "r"(v) : "memory"); }
SIMT_DEV void sts_v4(smem_ref r, uint32_t off, uint4 v) { asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(r.a + off), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory"); }
// shared-memory atomic add on an aligned 32-bit word, returns the old word (ATOMS.ADD)
SIMT_DEV uint32_t atoms_add(smem_ref r, uint32_t off, uint32_t v) { uint32_t o; asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(o) : "r"(r.a + off), "r"(v) : "memory"); return o; }

// Ampere-style asynchronous copy, 16 bytes global -> shared per lane (both addresses 16-byte aligned), tracked per thread:
// every lane of a warp copies for itself in ONE instruction (the bulk form, UBLKCP, takes uniform operands and would be
// serialised lane by lane).  commit closes the group of copies issued so far; wait<N> returns when all but the N most
// recent groups of the calling thread have landed.
SIMT_DEV void cp_async16(smem_ref r, uint32_t off, const void* g) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(r.a + off), "l"(g) : "memory"); }
SIMT_DEV void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> SIMT_DEV void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }
SIMT_DEV uint32_t atomic_inc(uint32_t* p) { return atomicAdd(p, 1u); }
SIMT_DEV uint32_t atomg_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }              // global memory, returns the old word
// load from L2, never from L1: for words that atomics modify (atomics are performed at L2; an L1 line filled by an earlier
// load of the same word would be stale)
SIMT_DEV uint32_t ldg_cg_u32(const uint32_t* p) { return __ldcg(p); }

// software prefetch of the line holding *p (no destination register, never faults the warp's progress)
SIMT_DEV void prefetch_l1(const void* p) { asm volatile("prefetch.global.L1 [%0];" :: "l"(p)); }
SIMT_DEV void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }

// ---- mbarrier + 1-D bulk async copy (global -> shared::cta), the TMA engine's non-tensor form --------------
struct mbar_t { uint64_t v; };

SIMT_DEV uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

SIMT_DEV void mbar_init(mbar_t* b, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(b)), "r"(count) : "memory");
}
SIMT_DEV void fence_mbar_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// one thread: arm the barrier phase with the total byte count of the copies that will complete_tx on it ...
SIMT_DEV void mbar_expect(mbar_t* b, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(b)), "r"(bytes) : "memory");
}
// ... then launch them (bytes: multiple of 16; both addresses 16 B aligned)
SIMT_DEV void bulk_copy(void* sdst, const void* gsrc, uint32_t bytes, mbar_t* b)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(sdst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(b)) : "memory");
}
SIMT_DEV void mbar_wait(mbar_t* b, uint32_t parity)
{
    uint32_t bar = smem_u32(b);
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" :: "r"(bar), "r"(parity) : "memory");
}

}  // namespace simt
#endif
