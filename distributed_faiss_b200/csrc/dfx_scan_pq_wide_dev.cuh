// dfx_scan_pq_wide_dev.cuh -- K3 + K4 for wide PQ codes, 64 < M <= 128 (included by
// dfx_search.cu; also compiled by the CPU emulator, tests/emu/).
//
// Replaces the inner loop of faiss IndexIVFPQ::search for shards with 65 to 128 sub-quantizers
// (reference index.py:43-48 with code_size > 64, or "IVF{n},PQ{M}" at index.py:385-396):
//   v = dis0 + (t + S),  S = halving-tree sum over P = 128 of lut[m][code_m] (oracle pq_sum,
//   positions m >= M hold +0).
// Reads the row-major codes (M bytes per vector), one lane per vector, like scan_pq_kernel; the probe
// loop, the walk and the candidate sink are the list-scan skeleton (dfx_scan_dev.cuh).
//
//   * The query's table, lut[m][j] = -2 * ip_seq(q_m, P[m][j]), is built in the prologue straight
//     into dynamic shared memory (M x 256 x 4 B: 96 KB at M = 96, 128 KB at M = 128).  A global
//     [queries][M][256] table would be 1 GiB per shard at the 8192-query chunk of the tensor-core
//     path; here the per-shard workspace is that of the other list scans (|q - c|^2 of the probes
//     and the per-group partial results).
//   * Registers: the first level of the tree adds position m and m + 64, so the lane forms
//     s[m] = lut[m][c_m] + lut[m+64][c_{m+64}] while it reads the codes (a literal +0.f where
//     m + 64 >= M, as the oracle's padding) and keeps 64 partials: the footprint of
//     scan_pq_kernel<64>.  dfx_halving_tree<32> then finishes the canonical order.
//   * The table lookups with random codes are not conflict-free (the bound of scan_pq_kernel too);
//     the row-major table is kept, so the arithmetic order is the oracle's without any remapping.
//   * THREADS (128 / 256 / 512) is chosen by the driver so that the table and one WarpTopK queue
//     per warp fit in the device's shared memory.
//   * MAT (k > 1024): the CTA's shared memory is the table only.
#pragma once
#include "dfx_common.cuh"
#include "dfx_scan_dev.cuh"

constexpr int PQW_KSUB = 256;
constexpr int PQW_MAX_M = 128;  // one query's fp32 table (M x 256 x 4 B) must fit in one CTA's shared memory

// shared memory of one CTA: the table, then the candidate queues
static inline size_t dfx_pq_wide_smem(int M, int threads, int cap, bool mat) {
    return (size_t)M * PQW_KSUB * 4 + dfx_scan_queue_smem(threads, cap, mat);
}

// MT: M when it is a multiple of 16 known at compile time (16-byte code loads), else 0 (any M % 4 == 0)
template <int MT, int THREADS, bool MAT = false>
__global__ void __launch_bounds__(THREADS)
scan_pq_wide_kernel(const float* __restrict__ Q, int d, int Mrt, int dsub, const float* __restrict__ codebooks,
                    const float* __restrict__ dis0, const int32_t* __restrict__ keys, int nprobe, int G,
                    int ngroups, const int64_t* __restrict__ list_off, const uint8_t* __restrict__ codes,
                    const float* __restrict__ tvals, const int32_t* __restrict__ ids, int k, int cap,
                    uint64_t* __restrict__ part, const int64_t* __restrict__ coff) {
    DFX_DYN_SMEM(unsigned char, smem_raw, 16);
    const int M = (MT > 0) ? MT : Mrt;
    float* s_lut = reinterpret_cast<float*>(smem_raw);  // [M][256]
    const ScanProbes pr(keys, dis0, list_off, nprobe, G, ngroups);

    // K3: entry e = m * 256 + j; a warp covers 32 consecutive j of one m (query loads are broadcasts,
    // codebook loads one contiguous run, table stores conflict-free).  seq-k order, as pq_prep_kernel.
    {
        const float* qrow = Q + pr.q * d;
#pragma unroll 4
        for (int e = threadIdx.x; e < M * PQW_KSUB; e += THREADS) {
            const float* qm = qrow + (e >> 8) * dsub;
            const float* p = codebooks + (size_t)e * dsub;
            float acc = 0.f;
            for (int t = 0; t < dsub; t++) acc = __fmaf_rn(__ldg(qm + t), __ldg(p + t), acc);
            s_lut[e] = -2.f * acc;
        }
    }
    ScanSink<MAT, THREADS> sink(reinterpret_cast<uint64_t*>(smem_raw + (size_t)M * PQW_KSUB * 4), cap, k, part,
                                coff);
    __syncthreads();

    dfx_scan_lanes<true>(pr, sink, [&](int64_t i, bool valid, int64_t, float d0) {
        float v = 0.f;
        uint32_t my_id = DFX_SEC_NONE;  // loaded with the code: never a dependent load on admission
        if (valid) {
            my_id = (uint32_t)__ldg(ids + i);
            float s[64];  // s[m] = lut[m][c_m] + lut[m + 64][c_{m+64}]: the tree's first level
            if (MT > 0) {
                static_assert(MT % 16 == 0, "MT must be a multiple of 16");
                const uint4* cp = reinterpret_cast<const uint4*>(codes + i * (int64_t)M);
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
                            const float a = s_lut[m * PQW_KSUB + ((wl[w] >> (8 * b)) & 255u)];
                            s[m] = hv ? a + s_lut[(m + 64) * PQW_KSUB + ((wh[w] >> (8 * b)) & 255u)] : a + 0.f;
                        }
                }
            } else {
                const uint32_t* cp = reinterpret_cast<const uint32_t*>(codes + i * (int64_t)M);
#pragma unroll
                for (int w = 0; w < 16; w++) {  // m = 4 w .. 4 w + 3
                    const bool hv = 4 * w + 64 < M;  // M % 4 == 0: the whole word is in or out
                    const uint32_t lo = __ldg(cp + w);
                    const uint32_t hi = hv ? __ldg(cp + 16 + w) : 0u;
#pragma unroll
                    for (int b = 0; b < 4; b++) {
                        const int m = 4 * w + b;
                        const float a = s_lut[m * PQW_KSUB + ((lo >> (8 * b)) & 255u)];
                        s[m] = hv ? a + s_lut[(m + 64) * PQW_KSUB + ((hi >> (8 * b)) & 255u)] : a + 0.f;
                    }
                }
            }
            dfx_halving_tree<32>(s);
            v = d0 + (__ldg(tvals + i) + s[0]);
        }
        return ScanCand{v, my_id};
    });
    // sink.finish(pr), but into row blockIdx.x (= q * ngroups + g) of `part`: keeping q and g live across
    // the scan costs 8 to 32 B more stack at 64 registers (DESIGN.md section 4.9)
    if constexpr (!MAT) cta_merge_and_write<THREADS>(sink.wt, sink.s_buf, cap, k, part + (int64_t)blockIdx.x * k);
}
