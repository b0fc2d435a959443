// dfx_scan_pq_fs_dev.cuh -- IVF-PQ FastScan (4-bit codes of the raw vectors, 8-bit quantized
// distance tables, integer sums; included by dfx_search.cu; also compiled by the CPU emulator, tests/emu/).
//
// Replaces the inner loop of faiss IndexIVFPQFastScan::search for shards described by the factory
// string "IVF{n},PQ{M}x4fs" (not by_residual).  The arithmetic is the canonical one of DESIGN.md
// section 2:
//   LUT[m][j]  = l2_seq(q_m, P[m][j])                              (fp32, as the encode)
//   mn_m = min_j LUT[m][j], span_m = max_j LUT[m][j] - mn_m
//   a = min(255 / max_m span_m, 65535 / sum_m span_m)  (a = 1 when every sub-table is flat)
//   b = sum_m mn_m                                     (sums over m ascending from +0)
//   LUTq[m][j] = floorf(fmaf(LUT[m][j] - mn_m, a, 0.5f))           (u8)
//   acc = sum_m LUTq[m][code_m]                                    (exact integer)
//   D = fmaf((float)acc, 1 / a, b)
// Candidates are ranked by (acc, id); the sum stays below 2^24, so (float)acc is exact and the
// ranking goes through the composites of the other list scans.
//
//   K_fs1 pq_fs_lut_kernel    one CTA per query: the fp32 table in shared memory, its quantization,
//                             LUTq u8[q][M][16] and (1 / a, b) to the workspace
//   K_fs2 scan_pq_fs_kernel   the list-scan skeleton (dfx_scan_dev.cuh), one lane per vector: the
//                             u8 table lives in M / 8 registers per lane
//   K_fs3 fs_dequant_kernel   the selected rows' D: (float)acc -> fmaf(acc, 1 / a, b); padding stays
#pragma once
#include "dfx_common.cuh"
#include "dfx_scan_dev.cuh"

// shared memory of pq_fs_lut_kernel: the query, the fp32 table, mn and span per sub-quantizer, a
static inline size_t dfx_pq_fs_lut_smem(int d, int M) { return (size_t)(d + M * 16 + 2 * M + 4) * 4; }

__global__ void __launch_bounds__(256)
pq_fs_lut_kernel(const float* __restrict__ Q, int d, int M, int dsub, const float* __restrict__ codebooks,
                 uint8_t* __restrict__ lutq, float2* __restrict__ qab) {
    DFX_DYN_SMEM(float, smem, 16);
    float* s_q = smem;                  // [d]
    float* s_lut = s_q + d;             // [M][16]
    float* s_mn = s_lut + M * 16;       // [M]
    float* s_span = s_mn + M;           // [M]
    float* s_a = s_span + M;            // [1]
    const int64_t q = blockIdx.x;
    const int tid = threadIdx.x;
    const int tot = M * 16;
    for (int i = tid; i < d; i += blockDim.x) s_q[i] = Q[q * d + i];
    __syncthreads();
    for (int idx = tid; idx < tot; idx += blockDim.x) {
        const float* p = codebooks + (size_t)idx * dsub;
        const float* qm = s_q + (idx >> 4) * dsub;
        float acc = 0.f;
        for (int t = 0; t < dsub; t++) {
            const float df = qm[t] - __ldg(p + t);
            acc = __fmaf_rn(df, df, acc);
        }
        s_lut[idx] = acc;
    }
    __syncthreads();
    for (int m = tid; m < M; m += blockDim.x) {
        float mn = s_lut[m * 16], mx = mn;
#pragma unroll
        for (int j = 1; j < 16; j++) {
            const float v = s_lut[m * 16 + j];
            mn = v < mn ? v : mn;
            mx = v > mx ? v : mx;
        }
        s_mn[m] = mn;
        s_span[m] = mx - mn;
    }
    __syncthreads();
    if (tid == 0) {  // M <= 128 sequential additions: the canonical order
        float span_max = 0.f, span_sum = 0.f, b = 0.f;
        for (int m = 0; m < M; m++) {
            const float s = s_span[m];
            span_max = s > span_max ? s : span_max;
            span_sum = span_sum + s;
            b = b + s_mn[m];
        }
        float a = 1.f;  // every sub-table flat: faiss divides by zero here; the value is pinned
        if (span_sum != 0.f) {
            const float a1 = dfx_div_rn(255.f, span_max), a2 = dfx_div_rn(65535.f, span_sum);
            a = a1 < a2 ? a1 : a2;
        }
        *s_a = a;
        qab[q] = make_float2(dfx_div_rn(1.f, a), b);
    }
    __syncthreads();
    const float a = *s_a;
    uint8_t* out = lutq + q * tot;
    for (int idx = tid; idx < tot; idx += blockDim.x)
        out[idx] = (uint8_t)(uint32_t)floorf(__fmaf_rn(s_lut[idx] - s_mn[idx >> 4], a, 0.5f));
}

//   * The table: lane L's word j holds LUTq[8j + 2c + (L >> 4)][L & 15] in byte c (c = 0..3), so one
//     SHFL of word m >> 3 from lane ((m & 1) << 4) | code_m returns LUTq[m][code_m] in byte
//     (m >> 1) & 3.  Byte c of word j is lutq[q][128 j + 32 c + L]: four coalesced byte loads.
//   * Code word j of a row (bytes 4j .. 4j + 3) holds the codes of sub-quantizers 8j .. 8j + 7, the
//     same ones as table word j; nibbles are split with the lane-half bit set as in K4n.
//   * The looked-up byte is masked in place and summed per byte position (acc_c += w & (0xff << 8c);
//     byte 3 is shifted down instead): at most M / 4 <= 32 terms per position, so no sum leaves
//     32 bits, and the four sums are folded once per vector.
//   * Tail lanes read the warp's first row, run every shuffle and are dropped at admission (as K4n).
//   * M = 72 and M >= 120: under ptxas's default register budget a few bytes spill to local memory;
//     asking for one resident block keeps everything in registers (72 to 96 of them).
template <int MT, bool MAT = false>
__global__ void __launch_bounds__(128, (MT == 72 || MT >= 120) ? 1 : 0)
scan_pq_fs_kernel(const uint8_t* __restrict__ lutq, const int32_t* __restrict__ keys, int nprobe, int G,
                  int ngroups, const int64_t* __restrict__ list_off, const uint8_t* __restrict__ codes,
                  const int32_t* __restrict__ ids, int k, int cap, uint64_t* __restrict__ part,
                  const int64_t* __restrict__ coff) {
    static_assert(MT >= 8 && MT <= 128 && MT % 8 == 0, "FastScan: M % 8 == 0, 8 <= M <= 128");
    constexpr int NW = MT / 8;  // 32-bit code words per row = 32-bit table words per lane
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    const ScanProbes pr(keys, nullptr, list_off, nprobe, G, ngroups);
    const int lane = threadIdx.x & 31;

    uint32_t T[NW];
    {
        const uint8_t* lq = lutq + pr.q * (int64_t)MT * 16 + lane;
#pragma unroll
        for (int j = 0; j < NW; j++)
            T[j] = (uint32_t)__ldg(lq + 128 * j) | ((uint32_t)__ldg(lq + 128 * j + 32) << 8) |
                   ((uint32_t)__ldg(lq + 128 * j + 64) << 16) | ((uint32_t)__ldg(lq + 128 * j + 96) << 24);
    }
    ScanSink<MAT, 128> sink(reinterpret_cast<uint64_t*>(smem_raw), cap, k, part, coff);

    dfx_scan_lanes<false>(pr, sink, [&](int64_t i, bool valid, int64_t base, float) {
        const int64_t r = valid ? i : base;  // tail lanes: the warp's first row
        uint32_t w[NW];
        dfx_load_code_words(codes + r * (MT / 2), w);
        const uint32_t my_id = (uint32_t)__ldg(ids + r);  // loaded with the codes: no dependent load on admission
        uint32_t acc0 = 0, acc1 = 0, acc2 = 0, acc3 = 0;
#pragma unroll
        for (int j = 0; j < NW; j++) {
            const uint32_t lo = w[j] & 0x0f0f0f0fu;
            const uint32_t hi = ((w[j] >> 4) & 0x0f0f0f0fu) | 0x10101010u;
            // sub-quantizers 8j + 2c + h: byte c of the code word and of the table word
            acc0 += __shfl_sync(0xffffffffu, T[j], (int)lo) & 0xffu;
            acc0 += __shfl_sync(0xffffffffu, T[j], (int)hi) & 0xffu;
            acc1 += __shfl_sync(0xffffffffu, T[j], (int)(lo >> 8)) & 0xff00u;
            acc1 += __shfl_sync(0xffffffffu, T[j], (int)(hi >> 8)) & 0xff00u;
            acc2 += __shfl_sync(0xffffffffu, T[j], (int)(lo >> 16)) & 0xff0000u;
            acc2 += __shfl_sync(0xffffffffu, T[j], (int)(hi >> 16)) & 0xff0000u;
            acc3 += __shfl_sync(0xffffffffu, T[j], (int)(lo >> 24)) >> 24;
            acc3 += __shfl_sync(0xffffffffu, T[j], (int)(hi >> 24)) >> 24;
        }
        // (float)acc, exact (acc <= 128 * 255 < 2^23), built as 2^23 + acc minus 2^23 rather than by
        // an I2F, which issues at an eighth of the FFMA rate on sm_90
        const uint32_t acc = acc0 + (acc1 >> 8) + (acc2 >> 16) + acc3;
        return ScanCand{__uint_as_float(0x4B000000u | acc) - 8388608.f, my_id};
    });
    sink.finish(pr);
}

// the selected rows of a query chunk: D = fmaf(acc, 1 / a, b) where an entry exists (I >= 0); the
// (+FLT_MAX, -1) padding is left as the selection wrote it
__global__ void fs_dequant_kernel(float* __restrict__ D, const int64_t* __restrict__ I, int64_t n, int k,
                                  const float2* __restrict__ qab) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || I[i] < 0) return;
    const float2 ab = qab[i / k];
    D[i] = __fmaf_rn(D[i], ab.x, ab.y);
}
