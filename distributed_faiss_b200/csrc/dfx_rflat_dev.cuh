// dfx_rflat_dev.cuh -- exact re-ranking on stored fp32 vectors (faiss IndexRefineFlat, the ",RFlat"
// suffix of a factory string).  Included by dfx_search.cu, whose driver launches it on the k'
// candidates the base kind's list scan selected.
//
// One warp per candidate.  A CTA of 8 warps takes 8 * U consecutive slots of ONE query's k'
// first-stage results (the grid is [query][ceil(k' / (8 U))]), so the query row is staged in shared
// memory once per CTA.  A candidate's row is addressed by its id directly: refine_vecs is in id
// order.  The distance is that of the IVF-Flat L2 scan (scan_rows_kernel MODE 1), bit for bit:
// lane j owns the dimensions 128 t + 4 j + u (u = 0..3), df = q_i - x_i, acc = fmaf(df, df, acc) in
// that order, then the butterfly xor 16 .. 1 (DESIGN.md section 2).  Each lane reads its part of the
// row with 16-byte loads; U = 2 candidates per warp are in flight for rows of up to 1 KB, where one
// row is at most two loads per lane and would leave the DRAM latency uncovered.  The composite
// (dis, id) goes to out[q * k1 + slot]; an empty slot (id -1) gives DFX_COMP_NONE.
#pragma once
#include "dfx_internal.h"

constexpr int RFLAT_WARPS = 8;  // warps per 256-thread CTA

template <int U>
__global__ void __launch_bounds__(32 * RFLAT_WARPS)
rflat_refine_kernel(const float* __restrict__ xq, int d, int k1, int ctas_per_query, const int64_t* __restrict__ cand,
                    const float* __restrict__ vecs, uint64_t* __restrict__ out) {
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    float* s_q = reinterpret_cast<float*>(smem_raw);
    const int64_t q = blockIdx.x / ctas_per_query;
    const int j0 = (blockIdx.x % ctas_per_query) * (RFLAT_WARPS * U) + (threadIdx.x >> 5) * U;
    const int lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < d; i += 32 * RFLAT_WARPS) s_q[i] = xq[q * d + i];
    __syncthreads();

    int64_t id[U];
    float acc[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
        id[u] = (j0 + u < k1) ? cand[q * k1 + j0 + u] : -1;
        acc[u] = 0.f;
    }
    for (int kb = 4 * lane; kb < d; kb += 128) {
        const float4 qv = *reinterpret_cast<const float4*>(s_q + kb);
        float4 xv[U];
#pragma unroll
        for (int u = 0; u < U; u++)
            xv[u] = (id[u] >= 0) ? __ldg(reinterpret_cast<const float4*>(vecs + id[u] * (int64_t)d + kb))
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int u = 0; u < U; u++) {
            float df;
            df = qv.x - xv[u].x; acc[u] = __fmaf_rn(df, df, acc[u]);
            df = qv.y - xv[u].y; acc[u] = __fmaf_rn(df, df, acc[u]);
            df = qv.z - xv[u].z; acc[u] = __fmaf_rn(df, df, acc[u]);
            df = qv.w - xv[u].w; acc[u] = __fmaf_rn(df, df, acc[u]);
        }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
        const float v = dfx_warp_butterfly(acc[u]);
        if (lane == 0 && j0 + u < k1)
            out[q * k1 + j0 + u] = (id[u] >= 0) ? dfx_comp(v, (uint32_t)id[u]) : DFX_COMP_NONE;
    }
}
