// dfx_pq_flat_dev.cuh -- product-quantized flat shards (FLAT_PQ: faiss IndexPQ(d, M, 8, metric), the
// factory string "PQ{M}"): the per-query distance table and the two kernels that score every stored
// code (included by dfx_search.cu; also compiled by the CPU emulator, tests/emu/).  DESIGN.md section 4.14.
//
//   pq_flat_lut_kernel     lut[q][m][j]: L2 l2_seq(q_m, P[m][j]), IP -ip_seq(q_m, P[m][j])
//   pq_flat_topk_kernel    k <= 100, or k <= 1024 with nq * k <= 16384 (pq_flat_fused): one CTA per (query,
//                          row tile), the tile's k best into its slot of the query's partial row (WarpTopK
//                          queues + cta_merge_and_write)
//   pq_flat_values_kernel  every other search and range search: the values of a column tile of flat_tiles,
//                          as gemm_values_kernel writes them for FLAT
// Both scoring kernels take a row's value from pq_flat_value, so the two paths agree bit for bit.
#pragma once
#include "dfx_common.cuh"
#include "dfx_topk.cuh"

constexpr int PQF_KSUB = 256;
constexpr int PQF_THREADS = 128;

// K3f: one CTA per query.  Entry e = m * 256 + j; t ascending from +0, the order of encode (L2).
__global__ void __launch_bounds__(256)
pq_flat_lut_kernel(const float* __restrict__ Q, int d, int M, int dsub, const float* __restrict__ codebooks,
                   int metric, float* __restrict__ lut) {
    const int64_t q = blockIdx.x;
    const float* qrow = Q + q * d;
    float* out = lut + q * (int64_t)M * PQF_KSUB;
    for (int e = threadIdx.x; e < M * PQF_KSUB; e += blockDim.x) {
        const float* qm = qrow + (e >> 8) * dsub;
        const float* p = codebooks + (size_t)e * dsub;
        float acc = 0.f;
        if (metric == DFX_METRIC_L2) {
            for (int t = 0; t < dsub; t++) {
                const float df = __ldg(qm + t) - __ldg(p + t);
                acc = __fmaf_rn(df, df, acc);
            }
        } else {
            for (int t = 0; t < dsub; t++) acc = __fmaf_rn(__ldg(qm + t), __ldg(p + t), acc);
            acc = -acc;
        }
        out[e] = acc;
    }
}

// The ranking value of code row `row` (M bytes, 4-byte aligned; 16-byte aligned when MT % 16 == 0):
// the halving tree over s_lut[m][code_m], positions m >= M holding +0.
//   !WIDE (M <= 64): P = MT for MT in {8, 16, 32, 64}, P = 64 for MT = 0 (any M % 4 == 0).
//   WIDE (64 < M <= 128): P = 128; the tree's first level, s[m] = lut[m][c_m] + lut[m + 64][c_{m+64}],
//   is formed while the codes are read, so a lane keeps 64 partials (scan_pq_wide_kernel's shape).
//   MT = 96 or 128 reads 16-byte words, MT = 0 32-bit words.
// Padding to 64 instead of the next power of two adds +0 where the shorter tree has nothing: it only
// turns a -0 into +0, which the composite key does as well.
template <int MT, bool WIDE>
__device__ __forceinline__ float pq_flat_value(const float* s_lut, const uint8_t* row, int M) {
    if constexpr (!WIDE) {
        constexpr int P = (MT > 0) ? MT : 64;
        float val[P];
        if constexpr (MT > 0 && (MT % 16) == 0) {
            const uint4* cp = reinterpret_cast<const uint4*>(row);
#pragma unroll
            for (int w4 = 0; w4 < MT / 16; w4++) {
                const uint4 c = __ldg(cp + w4);
                const uint32_t wv[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
                for (int w = 0; w < 4; w++) {
                    const int m = w4 * 16 + w * 4;
                    val[m + 0] = s_lut[(m + 0) * PQF_KSUB + (wv[w] & 255u)];
                    val[m + 1] = s_lut[(m + 1) * PQF_KSUB + ((wv[w] >> 8) & 255u)];
                    val[m + 2] = s_lut[(m + 2) * PQF_KSUB + ((wv[w] >> 16) & 255u)];
                    val[m + 3] = s_lut[(m + 3) * PQF_KSUB + (wv[w] >> 24)];
                }
            }
        } else {
            const uint32_t* cp = reinterpret_cast<const uint32_t*>(row);
#pragma unroll
            for (int w = 0; w < P / 4; w++) {
                const int m = w * 4;
                if (MT > 0 || m < M) {
                    const uint32_t c = __ldg(cp + w);
                    val[m + 0] = s_lut[(m + 0) * PQF_KSUB + (c & 255u)];
                    val[m + 1] = s_lut[(m + 1) * PQF_KSUB + ((c >> 8) & 255u)];
                    val[m + 2] = s_lut[(m + 2) * PQF_KSUB + ((c >> 16) & 255u)];
                    val[m + 3] = s_lut[(m + 3) * PQF_KSUB + (c >> 24)];
                } else {
                    val[m + 0] = val[m + 1] = val[m + 2] = val[m + 3] = 0.f;
                }
            }
        }
        dfx_halving_tree<P / 2>(val);
        return val[0];
    } else {
        float s[64];
        if constexpr (MT > 0) {
            static_assert(MT % 16 == 0 && MT > 64 && MT <= 128, "wide MT: a multiple of 16 in (64, 128]");
            const uint4* cp = reinterpret_cast<const uint4*>(row);
#pragma unroll
            for (int c = 0; c < 4; c++) {  // m = 16 c .. 16 c + 15
                constexpr int NH = (MT - 64) / 16;  // 16-code chunks of the upper half
                const bool hv = c < NH;
                const uint4 lo = __ldg(cp + c);
                const uint4 hi = hv ? __ldg(cp + 4 + c) : make_uint4(0u, 0u, 0u, 0u);
                const uint32_t wl[4] = {lo.x, lo.y, lo.z, lo.w};
                const uint32_t wh[4] = {hi.x, hi.y, hi.z, hi.w};
#pragma unroll
                for (int w = 0; w < 4; w++)
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        const int m = 16 * c + 4 * w + b;
                        const float a = s_lut[m * PQF_KSUB + ((wl[w] >> (8 * b)) & 255u)];
                        s[m] = hv ? a + s_lut[(m + 64) * PQF_KSUB + ((wh[w] >> (8 * b)) & 255u)] : a + 0.f;
                    }
            }
        } else {
            const uint32_t* cp = reinterpret_cast<const uint32_t*>(row);
#pragma unroll
            for (int w = 0; w < 16; w++) {  // m = 4 w .. 4 w + 3
                const bool hv = 4 * w + 64 < M;  // M % 4 == 0: the whole word is in or out
                const uint32_t lo = __ldg(cp + w);
                const uint32_t hi = hv ? __ldg(cp + 16 + w) : 0u;
#pragma unroll
                for (int b = 0; b < 4; b++) {
                    const int m = 4 * w + b;
                    const float a = s_lut[m * PQF_KSUB + ((lo >> (8 * b)) & 255u)];
                    s[m] = hv ? a + s_lut[(m + 64) * PQF_KSUB + ((hi >> (8 * b)) & 255u)] : a + 0.f;
                }
            }
        }
        dfx_halving_tree<32>(s);
        return s[0];
    }
}

// the query's table (lut [M][256] of query q) into shared memory
__device__ __forceinline__ void pq_flat_stage_lut(const float* __restrict__ lut, int64_t q, int M, float* s_lut) {
    const float4* src = reinterpret_cast<const float4*>(lut + q * (int64_t)M * PQF_KSUB);
    float4* dst = reinterpret_cast<float4*>(s_lut);
    for (int i = threadIdx.x; i < M * PQF_KSUB / 4; i += PQF_THREADS) dst[i] = src[i];
}

// K4f: blockIdx.x = t * qc + q (the chunk's queries run back to back over one tile, which then comes
// from L2).  Rows [t * tile, min(N, (t + 1) * tile)), one lane per row; the tile's k best (NONE padded)
// go to part[q * ld + t * k ..].  Shared memory: the table, then one queue of `cap` composites per warp.
template <int MT, bool WIDE>
__global__ void __launch_bounds__(PQF_THREADS)
pq_flat_topk_kernel(const float* __restrict__ lut, const uint8_t* __restrict__ codes, int64_t N, int64_t tile,
                    int qc, int Mrt, int k, int cap, uint64_t* __restrict__ part, int64_t ld) {
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    const int M = (MT > 0) ? MT : Mrt;
    const int64_t q = blockIdx.x % qc, t = blockIdx.x / qc;
    float* s_lut = reinterpret_cast<float*>(smem_raw);
    uint64_t* s_buf = reinterpret_cast<uint64_t*>(smem_raw + (size_t)M * PQF_KSUB * 4);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pq_flat_stage_lut(lut, q, M, s_lut);
    WarpTopK wt;
    wt.init(s_buf + (size_t)warp * cap, cap, k);
    __syncthreads();
    const int64_t beg = t * tile, end = min(N, beg + tile);
    for (int64_t base = beg + warp * 32; base < end; base += PQF_THREADS) {
        const int64_t i = base + lane;
        const bool valid = i < end;
        float v = 0.f;
        if (valid) v = pq_flat_value<MT, WIDE>(s_lut, codes + i * M, M);
        uint32_t sec = 0;
        const bool want = valid && wt.admits(v, [&] { return (uint32_t)i; }, sec);
        wt.push_lanes(want, v, sec);
    }
    cta_merge_and_write<PQF_THREADS>(wt, s_buf, cap, k, part + q * ld + t * k);
}

// K1f: the values of the nc rows from row c0 for the qc queries of a chunk, out[q * ld + j] = the value
// of row c0 + j (nc <= kFlatTile).  blockIdx.x = s * qc + q: query q, rows [s * span, min(nc, (s + 1) * span))
// of the tile.
// (4 resident CTAs requested: without it ptxas holds <96, true> to 40 registers and spills)
template <int MT, bool WIDE>
__global__ void __launch_bounds__(PQF_THREADS, 4)
pq_flat_values_kernel(const float* __restrict__ lut, const uint8_t* __restrict__ codes, int64_t c0, int nc, int span,
                      int qc, int Mrt, float* __restrict__ out, int64_t ld) {
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    const int M = (MT > 0) ? MT : Mrt;
    const int q = blockIdx.x % qc, s = blockIdx.x / qc;
    float* s_lut = reinterpret_cast<float*>(smem_raw);
    pq_flat_stage_lut(lut, q, M, s_lut);
    __syncthreads();
    const uint8_t* tc = codes + c0 * M;  // the tile's codes
    float* orow = out + q * ld;
    const int end = min(nc, (s + 1) * span);
    for (int j = s * span + threadIdx.x; j < end; j += PQF_THREADS)
        orow[j] = pq_flat_value<MT, WIDE>(s_lut, tc + (int64_t)j * M, M);
}
