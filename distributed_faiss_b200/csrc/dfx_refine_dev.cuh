// dfx_refine_dev.cuh -- IVF-PQR re-ranking (faiss IndexIVFPQR::search_preassigned's refinement).
// Included by dfx_search.cu, whose driver launches it on the k' candidates of the IVF-PQ stage.
//
// One warp per candidate (query q, slot j of the first stage's k' results): the candidate's id
// gives its storage position through `inv` and its list through a binary search of the list (or
// block) offsets, as reconstruct_kernel does.  The refined distance is
//     dis = sum_i (P2[m2][rcode_m2][.] - ((q_i - c_i) - P1[m1][code_m1][.]))^2
// in the warp-dot order of the IVF-Flat L2 scan: lane j owns the dimensions 128 t + 4 j + u
// (u = 0..3) and accumulates fmaf(df, df, acc) in that order, then the butterfly xor 16 .. 1
// (DESIGN.md section 2).  Each subtraction is one fp32 rounding.  The composite (dis, id) goes to
// out[c]; an empty slot (id -1) gives DFX_COMP_NONE.  Every table it reads (centroids, both
// codebooks, the codes) is small and L2-resident; nothing is staged in shared memory.
#pragma once
#include "dfx_internal.h"

constexpr int PQR_WARPS = 8;  // candidates per 256-thread CTA

// il != 0: `codes` are the interleaved blocks (dfx_il2_byte), `inv` holds padded block positions and
// `off` is blk_off; else `codes` are row-major u8[n][M] and `off` is list_off.
__global__ void __launch_bounds__(32 * PQR_WARPS)
pqr_refine_kernel(const float* __restrict__ xq, int d, int64_t ncand, int k1, const int64_t* __restrict__ cand,
                  const int32_t* __restrict__ inv, const int64_t* __restrict__ off, int64_t nlist, int il,
                  const uint8_t* __restrict__ codes, int M, int dsub, const float* __restrict__ cb1,
                  const uint8_t* __restrict__ rcodes, int M2, int dsub2, const float* __restrict__ cb2,
                  const float* __restrict__ cent, uint64_t* __restrict__ out) {
    const int64_t c = (int64_t)blockIdx.x * PQR_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (c >= ncand) return;  // warp-uniform
    const int64_t id = cand[c];
    if (id < 0) {
        if (lane == 0) out[c] = DFX_COMP_NONE;
        return;
    }
    const int64_t pos = inv[id];
    const int64_t l = dfx_list_of(off, nlist, il ? (pos >> 5) : pos);
    const float* q = xq + (c / k1) * d;
    const float* cl = cent + l * d;
    const uint8_t* rc = rcodes + id * M2;
    float acc = 0.f;
    for (int base = 4 * lane; base < d; base += 128) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int i = base + u;
            const int m = i / dsub, m2 = i / dsub2;
            const int code = il ? codes[(pos >> 5) * 1024 + dfx_il2_byte((int)(pos & 31), m)] : codes[pos * M + m];
            const float r1 = q[i] - cl[i];
            const float r2 = r1 - cb1[((size_t)m * 256 + code) * dsub + (i - m * dsub)];
            const float df = cb2[((size_t)m2 * 256 + rc[m2]) * dsub2 + (i - m2 * dsub2)] - r2;
            acc = __fmaf_rn(df, df, acc);
        }
    }
    acc = dfx_warp_butterfly(acc);
    if (lane == 0) out[c] = dfx_comp(acc, (uint32_t)id);
}
