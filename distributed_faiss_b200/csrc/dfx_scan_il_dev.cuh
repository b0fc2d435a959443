// dfx_scan_il_dev.cuh -- device code of dfx_scan_il.cu (also compiled by the CPU emulator, tests/emu/).
// Conversion between the row-major exchange form of an IVF-PQ shard (M == 32) and the 1 KB
// blocks of 32 vectors the scan reads (block layout: dfx_il2_byte, dfx_internal.h; scan kernel:
// dfx_scan_il2_dev.cuh).  Lists are padded to whole blocks; padding carries t = +inf so it can
// never enter a result.
#pragma once
#include "dfx_internal.h"
#include "dfx_topk.cuh"
#include "dfx_ptx.cuh"

// ------------------------------------------------------------------ layout conversion
// row-major (list-sorted) -> interleaved blocks.  one CTA per block.
__global__ void __launch_bounds__(256)
pq_rm_to_il_kernel(const int64_t* __restrict__ list_off, const int64_t* __restrict__ blk_off, int64_t nlist,
                   const uint8_t* __restrict__ codes, const float* __restrict__ tvals,
                   const int32_t* __restrict__ ids, uint8_t* __restrict__ il_codes, float* __restrict__ il_tvals,
                   int32_t* __restrict__ il_ids) {
    const int64_t blk = blockIdx.x;
    const int64_t l = dfx_list_of(blk_off, nlist, blk);
    const int64_t base = list_off[l] + (blk - blk_off[l]) * 32, end = list_off[l + 1];
    for (int e = threadIdx.x; e < 1024; e += 256) {
        const int v = e >> 5, m = e & 31;
        const int64_t i = base + v;
        il_codes[blk * 1024 + dfx_il2_byte(v, m)] = (i < end) ? codes[i * 32 + m] : (uint8_t)0;
    }
    if (threadIdx.x < 32) {
        const int64_t i = base + threadIdx.x;
        il_tvals[blk * 32 + threadIdx.x] = (i < end) ? tvals[i] : __int_as_float(0x7f800000);
        il_ids[blk * 32 + threadIdx.x] = (i < end) ? ids[i] : -1;
    }
}

__global__ void __launch_bounds__(256)
pq_il_to_rm_kernel(const int64_t* __restrict__ list_off, const int64_t* __restrict__ blk_off, int64_t nlist,
                   const uint8_t* __restrict__ il_codes, const float* __restrict__ il_tvals,
                   const int32_t* __restrict__ il_ids, uint8_t* __restrict__ codes, float* __restrict__ tvals,
                   int32_t* __restrict__ ids) {
    const int64_t blk = blockIdx.x;
    const int64_t l = dfx_list_of(blk_off, nlist, blk);
    const int64_t base = list_off[l] + (blk - blk_off[l]) * 32, end = list_off[l + 1];
    for (int e = threadIdx.x; e < 1024; e += 256) {
        const int v = e >> 5, m = e & 31;
        const int64_t i = base + v;
        if (i < end) codes[i * 32 + m] = il_codes[blk * 1024 + dfx_il2_byte(v, m)];
    }
    if (threadIdx.x < 32) {
        const int64_t i = base + threadIdx.x;
        if (i < end) {
            tvals[i] = il_tvals[blk * 32 + threadIdx.x];
            ids[i] = il_ids[blk * 32 + threadIdx.x];
        }
    }
}

