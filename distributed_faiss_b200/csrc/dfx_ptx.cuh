// dfx_ptx.cuh -- the inline-PTX primitives of the inverted-list scan kernels, in one place.
//
// Two implementations of each primitive: the PTX one (nvcc, sm_90a) and, under DFX_EMU, a plain
// C++ one used by the CPU lane-level emulator (tests/emu/): the emulator compiles the SAME
// kernel source with g++ and runs every CUDA thread as a fiber, so that the transcription of a
// kernel can be checked against the oracle without a GPU.  DFX_EMU is never defined in a
// product build.
#pragma once
#include <stdint.h>

// dynamic shared memory of the running kernel, as a typed pointer / array
#ifdef DFX_EMU
#define DFX_DYN_SMEM(type, name, align) type* name = reinterpret_cast<type*>(simt::dyn_smem())
#define DFX_DYN_SMEM0(type, name) type* name = reinterpret_cast<type*>(simt::dyn_smem())
#else
#define DFX_DYN_SMEM(type, name, align) extern __shared__ __align__(align) type name[]
#define DFX_DYN_SMEM0(type, name) extern __shared__ type name[]
#endif

// ---- streaming global loads: read once, do not allocate in L1
__device__ __forceinline__ uint4 dfx_ld_stream(const uint4* p) {
#ifdef DFX_EMU
    return *p;
#else
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
#endif
}
__device__ __forceinline__ float dfx_ld_stream_f(const float* p) {
#ifdef DFX_EMU
    return *p;
#else
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
#endif
}
// read-only global load that may stay in L1 (gathers)
__device__ __forceinline__ uint32_t dfx_ld_nc_u(const int32_t* p) {
#ifdef DFX_EMU
    return (uint32_t)*p;
#else
    uint32_t r;
    asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
#endif
}

// ---- shared memory by 32-bit shared-window address (see dfx_smem_addr)
// L2 prefetch of the 128-byte line holding p (no register result, no scoreboard)
__device__ __forceinline__ void dfx_prefetch_l2(const void* p) {
#ifndef DFX_EMU
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#else
    (void)p;
#endif
}

__device__ __forceinline__ uint32_t dfx_smem_addr(const void* p) {
#ifdef DFX_EMU
    return simt::smem_addr(p);
#else
    return (uint32_t)__cvta_generic_to_shared(p);
#endif
}
__device__ __forceinline__ float dfx_lds_f32(uint32_t addr) {
#ifdef DFX_EMU
    return *reinterpret_cast<const float*>(simt::smem_ptr(addr));
#else
    float r;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(r) : "r"(addr));
    return r;
#endif
}
