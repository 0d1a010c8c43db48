// hap_b200/csrc/simt.h
//
// The one header every kernel file includes.  Under nvcc it is just the CUDA runtime plus a launch
// macro.  Under HAPB200_EMU (tests/emu/, g++ only, never part of libhap_b200.so) it maps the CUDA
// execution model onto cooperative fibers so kernel logic can be unit-tested in a container without
// a GPU; that build is a development aid for tests only and is not a CPU fallback of the product.
#pragma once

#ifdef HAPB200_EMU
#include "simt_emu.h"
#else
#include <cuda_runtime.h>
#include <stdint.h>

#define HAP_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define HAP_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]

// Shared-memory accesses through a 32-bit shared-window address held in a register (for serial pointer-chasing
// loops: with generic addressing ptxas re-derives the window base -- an S2R -- in every iteration).
typedef uint32_t hap_saddr_t;
__device__ __forceinline__ hap_saddr_t hap_smem_addr(const void *p) { return (hap_saddr_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t hap_lds_u8(hap_saddr_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void hap_sts_u16(hap_saddr_t a, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" ::"r"(a), "h"((unsigned short)v)); }

// ---- sm_90 (Hopper) asynchronous bulk copies (TMA, 1-D) completed on an mbarrier ------------------------------------
// Global -> shared, `bytes` a multiple of 16, both addresses 16-byte aligned.  One thread issues the copy; the TMA unit
// moves the bytes without occupying issue slots or registers and signals the mbarrier with the byte count.
// SASS: UBLKCP (copy), SYNCS (mbarrier).  The emulator build (tests/emu/simt_emu.h) copies synchronously.
typedef unsigned long long hap_mbar_t;
__device__ __forceinline__ void hap_mbar_init(hap_mbar_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(hap_smem_addr(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void hap_mbar_expect_tx(hap_mbar_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(hap_smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void hap_tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, hap_mbar_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(hap_smem_addr(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(hap_smem_addr(bar))
                 : "memory");
}
// wait until the phase with the given parity has completed (HW-suspended wait, not a spin on memory)
__device__ __forceinline__ void hap_mbar_wait(hap_mbar_t *bar, uint32_t parity)
{
    uint32_t ok = 0;
    const hap_saddr_t a = hap_smem_addr(bar);
    do {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok)
                     : "r"(a), "r"(parity)
                     : "memory");
    } while (!ok);
}
// generic-proxy accesses to shared memory are ordered before later async-proxy (TMA) accesses
__device__ __forceinline__ void hap_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- device-scope flags between CTAs of one launch ------------------------------------------------------------------
__device__ __forceinline__ uint32_t hap_ld_acquire(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void hap_st_release(uint32_t *p, uint32_t v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void hap_nanosleep(uint32_t ns) { asm volatile("nanosleep.u32 %0;" ::"r"(ns)); }
#endif

#define HAP_FULL_MASK 0xffffffffu
